"""Pulses -> bits: the caller side of the digitizer (reference: ProtocolAnalyzer.get_protocol_from_signal
ProtocolAnalyzer.py:227-285 and _ppseq_to_bits :323-414).  Only what is needed to turn the pulse table into the bit
strings the reference's demodulation tests assert on; the protocol container / labels / decodings are out of scope.
The row loop runs on the GPU (bits.cu); its sequential CPU restatement lives in oracle/oracle.py (ppseq_to_bits), test-only."""
import array

import numpy as np

from ..cythonext import signal_functions


class LiteMessage(object):
    def __init__(self, bits, pause, bit_sample_pos, rssi=0.0):
        self.plain_bits = bits
        self.pause = pause
        self.bit_sample_pos = bit_sample_pos
        self.rssi = rssi

    @property
    def plain_bits_str(self) -> str:
        return "".join(map(str, self.plain_bits))

    def __len__(self):
        return len(self.plain_bits)


class ProtocolAnalyzer(object):
    def __init__(self, signal):
        self.signal = signal
        self.messages = []

    @property
    def plain_bits_str(self):
        return [m.plain_bits_str for m in self.messages]

    @property
    def plain_hex_str(self):
        out = []
        for m in self.messages:
            s = m.plain_bits_str
            s += "0" * ((4 - len(s) % 4) % 4)
            out.append("".join("{:x}".format(int(s[i:i + 4], 2)) for i in range(0, len(s), 4)))
        return out

    def get_protocol_from_signal(self):
        signal = self.signal
        self.messages = []
        if signal is None:
            return
        qad = signal.qad_device if hasattr(signal, "qad_device") else None
        if qad is None:   # no device copy (or one that would not fit): grab_pulse_lens streams the host qad when it must
            qad = signal.qad
        ppseq = signal_functions.grab_pulse_lens(
            qad, signal.center, signal.tolerance, signal.modulation_type, signal.samples_per_symbol,
            signal.bits_per_symbol, signal.center_spacing)
        bit_data, pauses, bit_sample_pos = self._ppseq_to_bits_device(
            ppseq, signal.samples_per_symbol, signal.bits_per_symbol, pause_threshold=signal.pause_threshold)
        if signal.message_length_divisor > 1 and signal.modulation_type == "ASK":
            self._ensure_message_length_multiple(bit_data, signal.samples_per_symbol, pauses, bit_sample_pos, signal.message_length_divisor)
        for i, (bits, pause) in enumerate(zip(bit_data, pauses)):
            middle = bit_sample_pos[i][int(len(bits) / 2)]
            rssi = np.mean(signal.iq_array.subarray(middle, middle + signal.samples_per_symbol).magnitudes_normalized)
            self.messages.append(LiteMessage(bits, pause, bit_sample_pos[i], rssi))

    # -- per-bit frequency estimation (ProtocolAnalyzer.py:416-447, 570-632; SURVEY 8f-4) -------------------------------------------
    def get_samplepos_of_bitseq(self, start_message: int, start_index: int, end_message: int, end_index: int, include_pause: bool):
        try:
            if start_message > end_message:
                start_message, end_message = end_message, start_message
            if start_index >= len(self.messages[start_message].bit_sample_pos) - 1:
                start_index = len(self.messages[start_message].bit_sample_pos) - 1
                if not include_pause:
                    start_index -= 1
            if end_index >= len(self.messages[end_message].bit_sample_pos) - 1:
                end_index = len(self.messages[end_message].bit_sample_pos) - 1
                if not include_pause:
                    end_index -= 1
            start = self.messages[start_message].bit_sample_pos[start_index]
            num_samples = self.messages[end_message].bit_sample_pos[end_index] - start
            return start, num_samples
        except (KeyError, IndexError):
            return -1, -1

    def estimate_frequency_for_one(self, sample_rate: float, nbits=42) -> float:
        return self.__estimate_frequency_for_bit(True, sample_rate, nbits)

    def estimate_frequency_for_zero(self, sample_rate: float, nbits=42) -> float:
        return self.__estimate_frequency_for_bit(False, sample_rate, nbits)

    def __estimate_frequency_for_bit(self, bit: bool, sample_rate: float, nbits: int) -> float:
        """mean of Signal.estimate_frequency (FFT arg-max on the device, urh_fft_argmax) over at most nbits bits equal to `bit`"""
        if nbits == 0:
            return 0
        assert self.signal is not None
        frequencies = []
        for i, message in enumerate(self.messages):
            for j, msg_bit in enumerate(message.plain_bits):
                if msg_bit == bit:
                    start, num_samples = self.get_samplepos_of_bitseq(i, j, i, j + 1, False)
                    frequencies.append(self.signal.estimate_frequency(start, start + num_samples, sample_rate))
                    if len(frequencies) == nbits:
                        return np.mean(frequencies)
        return np.mean(frequencies) if frequencies else 0

    @staticmethod
    def _ppseq_to_bits_device(ppseq, samples_per_symbol, bits_per_symbol, write_bit_sample_pos=True, pause_threshold=8):
        """_ppseq_to_bits with the row loop on the GPU (bits.cu); same return structure as the reference's."""
        bits, off, pause_arr, pos = signal_functions.ppseq_to_bits(ppseq, samples_per_symbol, bits_per_symbol, write_bit_sample_pos,
                                                                   pause_threshold)
        n_msgs = len(pause_arr)
        all_bits = [array.array("B", bits[off[m]:off[m + 1]].tobytes()) for m in range(n_msgs)]
        pauses = array.array("L", [int(v) for v in pause_arr])
        all_positions = []
        if write_bit_sample_pos:
            for m in range(n_msgs):
                lo = off[m] + 2 * m
                hi = min(off[m + 1] + 2 * m + 2, len(pos))
                all_positions.append(array.array("L", pos[lo:hi].astype(np.uint64).tobytes()))
        return all_bits, pauses, all_positions

    @staticmethod
    def _ensure_message_length_multiple(bit_data, samples_per_symbol, pauses, bit_sample_pos, divisor):
        for i in range(len(bit_data)):
            missing = (divisor - (len(bit_data[i]) % divisor)) % divisor
            if missing > 0 and pauses[i] >= samples_per_symbol * missing:
                bit_data[i].extend([0] * missing)
                pauses[i] = pauses[i] - missing * samples_per_symbol
                try:
                    bit_sample_pos[i][-1] = bit_sample_pos[i][-2] + samples_per_symbol
                except IndexError:
                    continue
                bit_sample_pos[i].extend([bit_sample_pos[i][-1] + (k + 1) * samples_per_symbol for k in range(missing - 1)])
                bit_sample_pos[i].append(bit_sample_pos[i][-1] + pauses[i])
