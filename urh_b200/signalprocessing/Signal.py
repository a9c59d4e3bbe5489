"""``Signal`` — a loaded capture and its demodulation parameters (reference: src/urh/signalprocessing/Signal.py).

Qt-free: the reference's pyqtSignals are plain callback lists here (``.connect`` / ``.emit`` keep working).
Same properties, cache-invalidation rules (``_qad = None`` on modulation type / bits per symbol / Costas bandwidth /
noise change) and methods; demodulation, noise detection, filtering and parameter estimation run on the GPU.
"""
import math
import os
import re
import tarfile
import tempfile
import wave

import numpy as np

from .. import _lib, settings
from ..ainterpretation import AutoInterpretation
from ..cythonext import signal_functions
from .Filter import Filter
from .IQArray import IQArray


class _Event(object):
    """stand-in for pyqtSignal: connect / disconnect / emit"""

    def __init__(self):
        self._slots = []

    def connect(self, fn):
        self._slots.append(fn)

    def disconnect(self, fn=None):
        self._slots = [s for s in self._slots if fn is not None and s is not fn]

    def emit(self, *args):
        for s in list(self._slots):
            s(*args)


class _Tracked(object):
    """One demodulation parameter of a Signal.  Assigning a DIFFERENT value stores it and then, as configured: drops the
    cached demodulation, fires ``<name>_changed`` with the new value, asks for a protocol update (unless updates are
    blocked).  Assigning the current value does nothing.  This is the reference's setter pattern (Signal.py:215-400),
    stated once instead of per property."""

    def __init__(self, cast=None, drops_qad=False, event=True, update=True):
        self.cast, self.drops_qad, self.event, self.update = cast, drops_qad, event, update

    def __set_name__(self, owner, name):
        self.name, self.slot = name, "_p_" + name

    def __get__(self, obj, owner=None):
        return self if obj is None else getattr(obj, self.slot)

    def __set__(self, obj, value):
        if self.cast is not None:
            value = self.cast(value)
        if getattr(obj, self.slot) == value:
            return
        setattr(obj, self.slot, value)
        if self.drops_qad:
            obj._drop_qad()
        if self.event:
            getattr(obj, self.name + "_changed").emit(value)
        if self.update:
            obj._needs_update()


class Signal(object):
    MODULATION_TYPES = ["ASK", "FSK", "PSK", "QAM"]
    _EVENTS = ("samples_per_symbol_changed", "tolerance_changed", "noise_threshold_changed", "center_changed",
               "center_spacing_changed", "name_changed", "sample_rate_changed", "modulation_type_changed",
               "bits_per_symbol_changed", "saved_status_changed", "protocol_needs_update", "data_edited")

    def __init__(self, filename: str, name="Signal", modulation: str = None, sample_rate: float = 1e6, timestamp: float = 0, parent=None):
        for e in self._EVENTS:
            setattr(self, e, _Event())
        # parameter slots are filled directly: construction fires no events
        defaults = dict(name=name, tolerance=5, samples_per_symbol=100, pause_threshold=8, message_length_divisor=1,
                        costas_loop_bandwidth=0.1, center=0, sample_rate=sample_rate, bits_per_symbol=1, center_spacing=1,
                        modulation_type="FSK" if modulation is None else modulation)
        for key, value in defaults.items():
            setattr(self, "_p_" + key, value)
        self._qad = None
        self._qad_dev = None
        self._noise_threshold = 0
        self.timestamp = timestamp
        self.noise_min_plot = 0
        self.noise_max_plot = 0
        self.block_protocol_update = False
        self.iq_array = IQArray(None, np.int8, 1)
        self.wav_mode = filename.endswith(".wav")
        self.flipper_raw_mode = filename.endswith(".sub")
        self.__changed = False
        self.parameter_cache = {mod: {"center": None, "samples_per_symbol": None} for mod in self.MODULATION_TYPES}
        self.__already_demodulated = False
        self.filename = ""
        if len(filename) > 0:
            if self.wav_mode:
                self.__load_wav_file(filename)
            elif self.flipper_raw_mode:
                self.__load_sub_file(filename)
            elif filename.endswith(".coco"):
                self.__load_compressed_complex(filename)
            else:
                self.iq_array = IQArray.from_file(filename)
            self.filename = filename
            default_noise_threshold = settings.read("default_noise_threshold", "automatic")
            if default_noise_threshold == "automatic":
                host = self.iq_array._peek()
                if AutoInterpretation.noise_level_streams(len(host), host.dtype,
                                                          signal_functions.device_budget(_lib.default_context())):
                    # the capture does not fit the device: streamed, and no device copy is kept
                    self.noise_threshold = AutoInterpretation.detect_noise_level_iq(host)
                else:
                    self.noise_threshold = AutoInterpretation.detect_noise_level_iq(self.iq_array.device())
            else:
                self.noise_threshold = float(default_noise_threshold) / 100 * self.max_magnitude

    # ---- loaders (Signal.py:114-213) -------------------------------------------------------------------------------
    def __load_wav_file(self, filename: str):
        wav = wave.open(filename, "r")
        num_channels, sample_width, sample_rate, num_frames, _, _ = wav.getparams()
        ranges = {1: (0, 255, np.uint8), 2: (-32768, 32767, np.int16), 3: (-8388608, 8388607, np.int32),
                  4: (-2147483648, 2147483647, np.int32)}
        if sample_width not in ranges:
            raise ValueError("Can't handle sample width {0}".format(sample_width))
        lo, hi, fmt = ranges[sample_width]
        mid = (lo + hi) / 2
        raw = wav.readframes(num_frames * num_channels)
        if sample_width == 3:
            count = len(raw) // (sample_width * num_channels)
            widened = np.empty((count, num_channels, 4), dtype=np.uint8)
            widened[:, :, :3] = np.frombuffer(raw, dtype=np.uint8).reshape(-1, num_channels, 3)
            widened[:, :, 3:] = (widened[:, :, 2:3] >> 7) * 255  # sign extension
            data = widened.view(np.int32).flatten()
        else:
            data = np.frombuffer(raw, dtype=fmt)
        self.iq_array = IQArray(None, np.float32, n=num_frames)
        if num_channels == 1:
            self.iq_array.real = np.multiply(1 / hi, np.subtract(data, mid))
            self.__already_demodulated = True
        elif num_channels == 2:
            self.iq_array.real = np.multiply(1 / hi, np.subtract(data[0::2], mid))
            self.iq_array.imag = np.multiply(1 / hi, np.subtract(data[1::2], mid))
        else:
            raise ValueError("Can't handle {0} channels. Only 1 and 2 are supported.".format(num_channels))
        wav.close()
        self.sample_rate = sample_rate

    def __load_sub_file(self, filename: str):
        # Flipper RAW (OOK): run lengths, positive = above center, negative = below
        hi, mid = 255, 127.5
        runs = []
        with open(filename, "r") as f:
            for line in f:
                m = re.match(r"RAW_Data:\s*([-0-9 ]+)\s*$", line)
                if not m:
                    continue
                for tok in m[1].strip().split(" "):
                    try:
                        v = int(tok)
                    except ValueError:
                        continue
                    runs.append(np.full(v, hi, dtype=np.uint8) if v > 0 else np.zeros(-v, dtype=np.uint8))
        arr = np.concatenate(runs) if runs else np.zeros(0, dtype=np.uint8)
        self.iq_array = IQArray(None, np.float32, n=len(arr))
        self.iq_array.real = np.multiply(1 / hi, np.subtract(arr, mid))
        self.__already_demodulated = True

    def __load_compressed_complex(self, filename: str):
        with tarfile.open(filename, "r") as tar:
            member = tar.getmembers()[0]
            tmpdir = tempfile.gettempdir()
            try:
                tar.extract(member, tmpdir, filter="data")
            except TypeError:
                tar.extract(member, tmpdir)
            path = os.path.join(tmpdir, tar.getnames()[0])
        self.iq_array = IQArray.from_file(path)
        os.remove(path)

    # ---- parameters (Signal.py:215-400) ----------------------------------------------------------------------------------
    # changing modulation type / bits per symbol / Costas bandwidth invalidates the demodulated samples; everything
    # but the name and the sample rate asks for a new protocol
    name = _Tracked(update=False)
    sample_rate = _Tracked(update=False)
    modulation_type = _Tracked(drops_qad=True)
    bits_per_symbol = _Tracked(cast=int, drops_qad=True)
    samples_per_symbol = _Tracked()
    tolerance = _Tracked(cast=int)
    center = _Tracked()
    center_spacing = _Tracked()
    pause_threshold = _Tracked(event=False)
    message_length_divisor = _Tracked(event=False)
    costas_loop_bandwidth = _Tracked(event=False, drops_qad=True)

    @property
    def already_demodulated(self) -> bool:
        return self.__already_demodulated

    def _needs_update(self):
        if not self.block_protocol_update:
            self.protocol_needs_update.emit()

    def _drop_qad(self):
        self._qad = None
        self._qad_dev = None

    @property
    def modulation_order(self):
        return 2 ** self.bits_per_symbol

    @property
    def center_thresholds(self):
        return self.get_thresholds_for_center(self.center)

    @property
    def num_samples(self):
        return self.iq_array.num_samples

    @property
    def noise_threshold(self):
        return self._noise_threshold

    @noise_threshold.setter
    def noise_threshold(self, value):
        if value != self.noise_threshold:
            self._drop_qad()
            self.clear_parameter_cache()
            self._noise_threshold = value
            middle = 0.5 * sum(IQArray.min_max_for_dtype(self.iq_array.dtype))
            a = self.max_amplitude * value / self.max_magnitude
            self.noise_min_plot = middle - a
            self.noise_max_plot = middle + a
            self.noise_threshold_changed.emit()
            self._needs_update()

    @property
    def max_magnitude(self):
        mi, ma = IQArray.min_max_for_dtype(self.iq_array.dtype)
        return (2 * max(mi ** 2, ma ** 2)) ** 0.5

    @property
    def max_amplitude(self):
        mi, ma = IQArray.min_max_for_dtype(self.iq_array.dtype)
        return 0.5 * (ma - mi)

    @property
    def noise_threshold_relative(self):
        return self.noise_threshold / self.max_magnitude

    @noise_threshold_relative.setter
    def noise_threshold_relative(self, value: float):
        self.noise_threshold = value * self.max_magnitude

    # ---- demodulation ---------------------------------------------------------------------------------------------------
    @property
    def qad_device(self):
        """demodulated samples resident in HBM (DeviceArray); feeds grab_pulse_lens without another upload.  None when the
        digitizer over a resident qad would not fit the device budget: grab_pulse_lens then streams the host qad."""
        q = self.qad  # demodulates on the GPU if necessary (and keeps the device copy)
        if self._qad_dev is None or len(self._qad_dev) != len(q):
            from ..device import to_device

            if signal_functions.use_stream(len(q), None, self.tolerance, _lib.STREAM_GRAB_PULSE_LENS,
                                           signal_functions.device_budget(_lib.default_context())):
                return None
            self._qad_dev = to_device(np.ascontiguousarray(q, dtype=np.float32))
        return self._qad_dev

    @property
    def qad(self):
        if self._qad is None:
            if self.already_demodulated:
                self._qad = np.ascontiguousarray(self.real_plot_data, dtype=self.real_plot_data.dtype)
            else:
                self._qad = self.quad_demod()
        return self._qad

    @property
    def real_plot_data(self):
        try:
            return self.iq_array.real
        except AttributeError:
            return np.zeros(0, dtype=np.float32)

    @property
    def imag_plot_data(self):
        try:
            return self.iq_array.imag
        except AttributeError:
            return np.zeros(0, dtype=np.float32)

    @property
    def real_plot_data_device(self):
        """`real_plot_data` resident in HBM (a DeviceColumn of `iq_array.device()`) for path_creator.create_path; reading it
        leaves the IQArray's device copy cached, which `real_plot_data` does not"""
        return self.iq_array.real_device

    @property
    def imag_plot_data_device(self):
        """`imag_plot_data` resident in HBM (see `real_plot_data_device`)"""
        return self.iq_array.imag_device

    @property
    def changed(self) -> bool:
        return self.__changed

    @changed.setter
    def changed(self, val: bool):
        if val != self.__changed:
            self.__changed = val
            self.saved_status_changed.emit()

    def _quad_demod_device(self):
        return signal_functions.afp_demod(self.iq_array.device(), self.noise_threshold, self.modulation_type,
                                          self.modulation_order, self.costas_loop_bandwidth)

    def _host_capture_too_large(self):
        """the host capture when demodulating it resident would exceed the device budget and it can be streamed instead (ASK /
        FSK / PSK; a capture already on the device fits), else None"""
        iq = self.iq_array
        if self.modulation_type not in ("ASK", "FSK", "PSK") or iq._device is not None or len(iq) <= 2:
            return None
        host = iq._peek()
        entry = _lib.STREAM_AFP_DEMOD
        if self.modulation_type == "PSK":   # the Costas loop's tables grow with the loop order
            entry |= signal_functions.psk_entry(self.modulation_order)
        if not signal_functions.use_stream(len(host), host.dtype, 0, entry, signal_functions.device_budget(_lib.default_context())):
            return None
        return host

    def quad_demod(self):
        if self.noise_threshold < self.max_magnitude:
            host = self._host_capture_too_large()
            if host is not None:   # streamed through the device: qad comes back to the host, nothing stays resident
                self._qad_dev = None
                return signal_functions.afp_demod(host, self.noise_threshold, self.modulation_type, self.modulation_order,
                                                  self.costas_loop_bandwidth)
            self._qad_dev = self._quad_demod_device()
            return self._qad_dev.get()
        return np.zeros(2, dtype=np.float32)

    def calc_relative_noise_threshold_from_range(self, noise_start: int, noise_end: int):
        noise_start, noise_end = int(noise_start), int(noise_end)
        if noise_start > noise_end:
            noise_start, noise_end = noise_end, noise_start
        try:
            maximum = np.max(self.iq_array.subarray(noise_start, noise_end).magnitudes_normalized)
            return np.ceil(maximum * 10 ** 4) / 10 ** 4
        except ValueError:
            return self.noise_threshold_relative

    def create_new(self, start=0, end=0, new_data=None, new_timestamp=0):
        new_signal = Signal("", "New " + self.name)
        if new_data is None:
            new_signal.iq_array = IQArray(np.array(self.iq_array._peek(slice(start, end)), order="C"), _owned=True)
            new_signal.timestamp = self.timestamp + (start / self.sample_rate)
        else:
            new_signal.iq_array = IQArray(new_data)
            new_signal.timestamp = new_timestamp
        new_signal._noise_threshold = self.noise_threshold
        new_signal.noise_min_plot = self.noise_min_plot
        new_signal.noise_max_plot = self.noise_max_plot
        new_signal._p_samples_per_symbol = self.samples_per_symbol
        new_signal._p_bits_per_symbol = self.bits_per_symbol
        new_signal._p_center = self.center
        new_signal.wav_mode = self.wav_mode
        new_signal.flipper_raw_mode = self.flipper_raw_mode
        new_signal._Signal__already_demodulated = self.already_demodulated
        new_signal.changed = True
        new_signal.sample_rate = self.sample_rate
        return new_signal

    def get_thresholds_for_center(self, center: float, spacing=None):
        spacing = self.center_spacing if spacing is None else spacing
        return signal_functions.get_center_thresholds(center, spacing, self.modulation_order)

    def auto_detect(self, emit_update=True, detect_modulation=True, detect_noise=False) -> bool:
        kwargs = {
            "noise": None if detect_noise else self.noise_threshold,
            "modulation": None if detect_modulation
            else "OOK" if self.bits_per_symbol == 1 and self.modulation_type == "ASK" else self.modulation_type,
        }
        estimated = AutoInterpretation.estimate(self.iq_array, **kwargs)
        if estimated is None:
            return False
        orig_block = self.block_protocol_update
        self.block_protocol_update = True
        if detect_noise:
            self.noise_threshold = estimated["noise"]
        if detect_modulation:
            self.modulation_type = estimated["modulation_type"]
        self.center = estimated["center"]
        self.tolerance = estimated["tolerance"]
        self.samples_per_symbol = estimated["bit_length"]
        self.block_protocol_update = orig_block
        if emit_update and not self.block_protocol_update:
            self.protocol_needs_update.emit()
        return True

    def clear_parameter_cache(self):
        for mod in self.parameter_cache.keys():
            self.parameter_cache[mod]["samples_per_symbol"] = None
            self.parameter_cache[mod]["center"] = None

    def estimate_frequency(self, start: int, end: int, sample_rate: float):
        """FFT arg-max of a power-of-two window (Signal.py:578-601); transform and arg-max on the GPU (modulation.cu)"""
        import ctypes as C

        from .. import _lib
        from ..device import to_device

        if end - start <= 0:
            return 100e3  # empty window
        length = 2 ** int(math.log2(end - start))
        data = np.ascontiguousarray(self.iq_array.as_complex64()[start: start + length])
        if len(data) == 0:
            return 100e3
        ctx = _lib.default_context()
        d = to_device(data.view(np.float32), ctx)
        idx, P = C.c_int64(0), C.c_int64(0)
        ctx.check(ctx.lib.urh_fft_argmax(ctx.handle, C.c_void_p(d.ptr), len(data), C.byref(idx), C.byref(P)))
        n = P.value
        k = idx.value
        freq = (k if k < (n + 1) // 2 else k - n) / n   # np.fft.fftfreq(n)[k]
        return abs(freq * sample_rate)

    def eliminate(self):
        self.iq_array = None
        self._drop_qad()
        self.parameter_cache.clear()

    def silent_set_modulation_type(self, mod_type: str):
        self._p_modulation_type = mod_type

    # ---- edit operations (Signal.py:613-651) --------------------------------------------------------------------------------
    def insert_data(self, index: int, data: np.ndarray):
        self.iq_array.insert_subarray(index, data)
        self._drop_qad()
        self.__invalidate_after_edit()

    def delete_range(self, start: int, end: int):
        mask = np.ones(self.num_samples, dtype=bool)
        mask[start:end] = False
        try:
            self.iq_array.apply_mask(mask)
            self._qad = self._qad[mask] if self._qad is not None else None
            self._qad_dev = None
        except IndexError:
            pass
        self.__invalidate_after_edit()

    def mute_range(self, start: int, end: int):
        self.iq_array[start:end] = 0
        if self._qad is not None:
            self._qad[start:end] = 0
        self._qad_dev = None
        self.__invalidate_after_edit()

    def crop_to_range(self, start: int, end: int):
        self.iq_array = IQArray(np.array(self.iq_array._peek(slice(start, end)), order="C"), _owned=True)
        self._qad = self._qad[start:end] if self._qad is not None else None
        self._qad_dev = None
        self.__invalidate_after_edit()

    def filter_range(self, start: int, end: int, fir_filter: Filter):
        self.iq_array[start:end] = fir_filter.work(self.iq_array[start:end])
        self._qad[start:end] = signal_functions.afp_demod(
            np.ascontiguousarray(self.iq_array[start:end]), self.noise_threshold, self.modulation_type, self.modulation_order,
            self.costas_loop_bandwidth)
        self._qad_dev = None
        self.__invalidate_after_edit()

    def __invalidate_after_edit(self):
        self.clear_parameter_cache()
        self.changed = True
        self.data_edited.emit()
        self.protocol_needs_update.emit()

    @staticmethod
    def from_samples(samples: np.ndarray, name: str, sample_rate: float):
        signal = Signal("", name, sample_rate=sample_rate)
        signal.iq_array = IQArray(samples)
        return signal
