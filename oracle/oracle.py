"""Python face of the CPU oracle.  TEST INFRASTRUCTURE ONLY (see urh_oracle.c header).

* C restatement (liburh_oracle.so): afp_demod, grab_pulse_lens, get_magnitudes, segment_messages,
  fir_filter, arr2decibel, modulate, median_filter, plateau_lengths.
* numpy restatements of the reference's Python-level DSP (AutoInterpretation.detect_noise_level /
  detect_center, Spectrogram.stft, Filter bandpass design, gauss_fir, ...), each citing file:line.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this module.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liburh_oracle.so")

DT = {np.dtype(np.int8): 0, np.dtype(np.uint8): 1, np.dtype(np.int16): 2, np.dtype(np.uint16): 3, np.dtype(np.float32): 4}
MOD = {"ASK": 0, "FSK": 1, "PSK": 2, "QAM": 3, "GFSK": 4, "OQPSK": 5}

_lib = None


def build(force=False):
    src = os.path.join(HERE, "urh_oracle.c")
    if force or not os.path.isfile(LIB) or os.path.getmtime(LIB) < os.path.getmtime(src):
        subprocess.check_call(
            ["/usr/bin/gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
             "-o", LIB, src, "-lm"]
        )
    return LIB


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
        _lib.oracle_grab_pulse_lens.restype = C.c_int64
        _lib.oracle_segment_messages.restype = C.c_int64
        _lib.oracle_plateau_lengths.restype = C.c_int64
        _lib.oracle_noise_value.restype = C.c_float
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def afp_demod(samples, noise_mag, mod_type, mod_order, costas_loop_bandwidth=0.1):
    samples = np.ascontiguousarray(samples)
    n = len(samples)
    out = np.zeros(n, dtype=np.float32)
    rc = lib().oracle_afp_demod(_p(samples), DT[samples.dtype], C.c_int64(n), C.c_float(noise_mag), MOD.get(mod_type, 99),
                                int(mod_order), C.c_float(costas_loop_bandwidth), _p(out))
    if rc != 0:
        raise ValueError("Unsupported dtype")
    return out


def costas_from(samples, noise_mag, loop_order, state, costas_loop_bandwidth=0.1):
    """The Costas loop (signal_functions.pyx:289-328) over ALL of `samples`, continued from the loop state (freq, phase) a
    preceding segment ended in -> (demodulated float32, end state).  Checker for captures sharded over GPUs."""
    samples = np.ascontiguousarray(samples)
    n = len(samples)
    out = np.zeros(n, dtype=np.float32)
    end = np.zeros(2, dtype=np.float32)
    lib().oracle_costas_from(_p(samples), DT[samples.dtype], C.c_int64(n), C.c_float(noise_mag), int(loop_order),
                             C.c_float(costas_loop_bandwidth), C.c_float(state[0]), C.c_float(state[1]), _p(out), _p(end))
    return out, end


def get_center_thresholds(center, spacing, order):
    out = np.empty(max(order - 1, 0), dtype=np.float32)
    lib().oracle_center_thresholds(C.c_float(center), C.c_float(spacing), int(order), _p(out))
    return out


def grab_pulse_lens(samples, center, tolerance, modulation_type, samples_per_symbol, bits_per_symbol=1, center_spacing=0.1):
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    n = len(samples)
    rows = np.zeros((max(n, 1), 2), dtype=np.int64)
    k = lib().oracle_grab_pulse_lens(_p(samples), C.c_int64(n), C.c_float(center), C.c_uint16(tolerance),
                                     MOD.get(modulation_type, 99), C.c_uint32(samples_per_symbol),
                                     C.c_uint8(bits_per_symbol), C.c_float(center_spacing), _p(rows))
    return rows[:k].copy()


def get_magnitudes(iq):
    iq = np.ascontiguousarray(iq)
    out = np.zeros(len(iq), dtype=np.float64)
    lib().oracle_get_magnitudes(_p(iq), DT[iq.dtype], C.c_int64(len(iq)), _p(out))
    return out


def segment_messages_from_magnitudes(mags, noise_threshold):
    mags = np.ascontiguousarray(mags)
    assert mags.dtype in (np.float32, np.float64)
    out = np.zeros((len(mags) // 10 + 2, 2), dtype=np.int64)
    k = lib().oracle_segment_messages(_p(mags), int(mags.dtype == np.float64), C.c_int64(len(mags)),
                                      C.c_float(noise_threshold), _p(out))
    return [(int(a), int(b)) for a, b in out[:k]]


def fir_filter(x, taps):
    x = np.ascontiguousarray(x, dtype=np.complex64)
    taps = np.ascontiguousarray(taps, dtype=np.complex64)
    # the reference's shape, np.zeros(N + M - 1)[:N]: N - 1 outputs without taps, ValueError (negative dimensions) for N = M = 0
    shape = np.zeros(len(x) + len(taps) - 1, dtype=np.complex64)[: len(x)].shape
    out = np.zeros(len(x), dtype=np.complex64)
    lib().oracle_fir_filter(_p(x), C.c_int64(len(x)), _p(taps), C.c_int64(len(taps)), _p(out))
    return out[: shape[0]]


def arr2decibel(arr):
    arr = np.ascontiguousarray(arr, dtype=np.complex64)
    out = np.empty(arr.shape, dtype=np.float32)
    lib().oracle_arr2decibel(_p(arr), C.c_int64(arr.size), _p(out))
    return out


def median_filter(data, k=3):
    data = np.ascontiguousarray(data, dtype=np.float64)
    out = np.zeros(len(data), dtype=np.float32)
    lib().oracle_median_filter(_p(data), C.c_int64(len(data)), C.c_uint(k), _p(out))
    return out


def get_plateau_lengths(rect, center, percentage=25):
    rect = np.ascontiguousarray(rect, dtype=np.float32)
    if len(rect) == 0 or center is None:
        return np.array([], dtype=np.uint64)
    out = np.zeros(len(rect), dtype=np.uint64)
    k = lib().oracle_plateau_lengths(_p(rect), C.c_int64(len(rect)), C.c_float(center), int(percentage), _p(out))
    return out[:k].copy()


# ---- modulator ---------------------------------------------------------------------------------------
def gauss_fir(sample_rate, samples_per_symbol, bt=0.5, filter_width=1.0):
    """signal_functions.pyx:228-243 (float32 arithmetic as numpy evaluates it)."""
    sample_rate = np.float32(sample_rate)
    bt = np.float32(bt)
    filter_width = np.float32(filter_width)
    k = np.arange(-int(filter_width * samples_per_symbol), int(filter_width * samples_per_symbol) + 1, dtype=np.float32)
    ts = np.float32(np.float32(samples_per_symbol) / sample_rate)
    h = (np.sqrt((2 * np.pi) / (np.log(2))) * bt / ts * np.exp(
        -(((np.sqrt(2) * np.pi) / np.sqrt(np.log(2)) * bt * k / samples_per_symbol) ** 2))).astype(np.float32)
    return h / h.sum()


def gauss_filtered_freqs_phases(bits, parameters, num_symbols, sps, sample_rate, phi, start, gauss_bt, filter_width):
    """signal_functions.pyx:196-226."""
    bits = np.asarray(bits, dtype=np.uint8)
    bps = int(len(bits) // num_symbols)
    weights = 1 << np.arange(bps - 1, -1, -1)
    idx = (bits[: num_symbols * bps].reshape(num_symbols, bps) * weights).sum(axis=1)
    frequencies = np.repeat(np.asarray(parameters, dtype=np.float32)[idx], sps).astype(np.float32)
    num_values = num_symbols * sps
    t = np.arange(start, start + num_values, dtype=np.float32) / np.float32(sample_rate)
    gfir = gauss_fir(sample_rate, sps, bt=gauss_bt, filter_width=filter_width)
    if len(frequencies) >= len(gfir):
        frequencies = np.convolve(frequencies, gfir, mode="same")
    else:
        frequencies = np.convolve(gfir, frequencies, mode="same")[: len(frequencies)]
    frequencies = frequencies.astype(np.float32)
    phases = np.zeros(len(frequencies), dtype=np.float32)
    phases[0] = phi
    two_pi = 2 * math.pi
    # serial float32-rounded recurrence, double arithmetic inside (pyx:222-224)
    ph = float(np.float32(phi))
    tt = t.astype(np.float64)
    df = frequencies[:-1].astype(np.float64) - frequencies[1:].astype(np.float64)
    # frequencies[i] - frequencies[i+1] is a float32 subtraction in the reference (both float32 ndarray elements)
    df32 = (frequencies[:-1] - frequencies[1:]).astype(np.float64)
    del df
    for i in range(len(phases) - 1):
        ph = float(np.float32(two_pi * tt[i] * df32[i] + ph))
        phases[i + 1] = ph
    return np.column_stack((frequencies, phases)).astype(np.float32)


def get_oqpsk_bits(bits):
    """signal_functions.pyx:179-193."""
    bits = np.asarray(bits, dtype=np.uint8)
    n = len(bits)
    if n == 0:
        return np.zeros(0, dtype=np.uint8)
    r = np.zeros(n + 2, dtype=np.uint8)
    r[0] = bits[0]
    r[n + 1] = bits[n - 1]
    for i in range(2, n - 2, 2):
        r[i] = bits[i]
        r[i + 1] = bits[i - 1]
    return r


def modulate_c(bits, samples_per_symbol, modulation_type, parameters, bits_per_symbol, carrier_amplitude,
               carrier_frequency, carrier_phase, sample_rate, pause, start, dtype=np.float32, gauss_bt=0.5, filter_width=1.0,
               gfsk_table=None):
    """signal_functions.pyx:56-177.  gfsk_table: a (symbols * sps, 2) float32 (frequency, phase) table to modulate GFSK from
    instead of gauss_filtered_freqs_phases (checks the sample stage of a GPU table)."""
    bits = np.ascontiguousarray(np.asarray(bits, dtype=np.uint8))
    params = np.ascontiguousarray(np.asarray(parameters, dtype=np.float32))
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype(np.int8), np.dtype(np.int16), np.dtype(np.float32)):
        raise ValueError("Unsupported dtype for modulation {}".format(dtype))
    num_bits = len(bits)
    total_symbols = int(num_bits // bits_per_symbol)
    total = total_symbols * samples_per_symbol + pause
    out = np.zeros((total, 2), dtype=dtype)
    if num_bits == 0:
        return out
    mod = modulation_type.upper()
    assert mod in ("FSK", "ASK", "PSK", "GFSK", "OQPSK")
    gtab = None
    if mod == "OQPSK":
        assert bits_per_symbol == 2
        bits = np.ascontiguousarray(get_oqpsk_bits(bits))
    if mod == "GFSK" and gfsk_table is not None:
        gtab = np.ascontiguousarray(gfsk_table, dtype=np.float32)
        assert gtab.shape == (total_symbols * samples_per_symbol, 2), gtab.shape
    elif mod == "GFSK":
        gtab = np.ascontiguousarray(gauss_filtered_freqs_phases(bits, params, total_symbols, samples_per_symbol,
                                                                sample_rate, carrier_phase, start, gauss_bt, filter_width))
    lib().oracle_modulate(_p(bits), C.c_int64(num_bits), C.c_uint32(samples_per_symbol), MOD[mod], _p(params),
                          C.c_uint16(bits_per_symbol), C.c_float(carrier_amplitude), C.c_float(carrier_frequency),
                          C.c_float(carrier_phase), C.c_float(sample_rate), C.c_uint32(pause), C.c_uint32(start),
                          DT[dtype], _p(gtab) if gtab is not None else None, _p(out))
    return out


# ---- AutoInterpretation (numpy level) -----------------------------------------------------------------
def minmax(arr):
    """util.pyx:20-36"""
    if len(arr) == 0:
        return 0, 0
    # the Cython function returns C scalars converted to Python numbers (float32 -> Python float)
    return arr.min().item(), arr.max().item()


def detect_noise_level(magnitudes):
    """AutoInterpretation.py:60-91"""
    if len(magnitudes) <= 3:
        return 0
    chunksize = max(1, int(len(magnitudes) * 1 / 100))
    chunks = [magnitudes[i - chunksize: i] for i in range(len(magnitudes), 0, -chunksize) if i - chunksize >= 0]
    mean_values = np.fromiter((np.mean(chunk) for chunk in chunks), dtype=np.float32, count=len(chunks))
    minimum, maximum = minmax(mean_values)
    if maximum == 0 or minimum / maximum > 0.9:
        return 0
    indices = np.nonzero(mean_values <= 1.1 * np.min(mean_values))[0]
    try:
        result = np.max([np.max(chunks[i]) for i in indices if len(chunks[i]) > 0])
    except ValueError:
        return 0
    return math.ceil(result * 10000) / 10000


def detect_center(rectangular_signal, max_size=None):
    """AutoInterpretation.py:226-277"""
    rect = rectangular_signal[rectangular_signal > -4]
    rect = rect[int(0.05 * len(rect)): int(0.95 * len(rect))]
    if max_size is not None and len(rect) > max_size:
        rect = rect[0:max_size]
    hist_min, hist_max = minmax(rect)
    hist_step = float(np.var(rect))
    try:
        y, x = np.histogram(rect, bins=np.arange(hist_min, hist_max + hist_step, hist_step))
    except (ZeroDivisionError, ValueError):
        return None
    most_common_levels = []
    window_size = max(2, int(0.05 * len(y)) + 1)

    def get_elem(arr, index, default):
        return arr[index] if 0 <= index < len(arr) else default

    for index in np.argsort(y)[::-1]:
        if all(y[index] > get_elem(y, index + i, 0) and y[index] > get_elem(y, index - i, 0) for i in range(1, window_size)):
            most_common_levels.append(x[index])
        if len(most_common_levels) == 2:
            break
    if len(most_common_levels) == 0:
        return None
    return np.mean(most_common_levels)


# ---- Spectrogram / Filter (numpy level) -----------------------------------------------------------------
def stft(samples, window_size=1024, overlap_factor=0.5, window_function=np.hanning):
    """Spectrogram.py:94-116"""
    window = window_function(window_size)
    hop = window_size - int(overlap_factor * window_size)
    if len(samples) < window_size:
        samples = np.append(samples, np.zeros(window_size - len(samples)))
    num_frames = max(1, (len(samples) - window_size) // hop + 1)
    shape = (num_frames, window_size)
    strides = (hop * samples.strides[-1], samples.strides[-1])
    frames = np.lib.stride_tricks.as_strided(samples, shape=shape, strides=strides)
    return np.fft.fft(frames * window, window_size) / np.atleast_1d(window_size)


def spectrogram_db(samples, window_size=1024, overlap_factor=0.5, window_function=np.hanning):
    """Spectrogram.py:156-162"""
    spec = np.fft.fftshift(stft(samples, window_size, overlap_factor, window_function), axes=(1,))
    return np.fliplr(arr2decibel(spec.astype(np.complex64)))


def filter_length_from_bandwidth(bw):
    """Filter.py:64-67"""
    N = int(math.ceil(4 / bw))
    return N + 1 if N % 2 == 0 else N


def design_windowed_sinc_lpf(fc, bw):
    """Filter.py:103-119"""
    N = filter_length_from_bandwidth(bw)
    h = np.sinc(2 * fc * (np.arange(N) - (N - 1) / 2.0))
    h = h * np.blackman(N)
    return h / np.sum(h)


def design_windowed_sinc_bandpass(f_low, f_high, bw):
    """Filter.py:121-131"""
    f_shift = (f_low + f_high) / 2
    f_c = (f_high - f_low) / 2
    N = filter_length_from_bandwidth(bw)
    return design_windowed_sinc_lpf(f_c, bw=bw) * np.exp(complex(0, 1) * np.pi * 2 * f_shift * np.arange(0, N, dtype=complex))


def fft_convolve_1d(x, h):
    """Filter.py:69-82: complex transforms when x or h is complex, else rfft / irfft (a real result)"""
    n = len(x) + len(h) - 1
    n_opt = 1 << (n - 1).bit_length()
    if np.iscomplexobj(x) or np.iscomplexobj(h):
        fft, ifft = np.fft.fft, np.fft.ifft
    else:
        fft, ifft = np.fft.rfft, np.fft.irfft
    result = ifft(fft(x, n_opt) * fft(h, n_opt), n_opt)[0:n]
    too_much = (len(result) - len(x)) // 2
    return result[too_much:-too_much]


def dc_correction(x):
    """Filter.py:31-33 (Filter.work with FilterType.dc_correction)"""
    return x - np.mean(x, axis=0)


def apply_bandpass_filter(data, f_low, f_high, filter_bw=0.08):
    """Filter.py:84-101"""
    if f_low > f_high:
        f_low, f_high = f_high, f_low
    f_low = max(-0.5, min(0.5, f_low))
    f_high = max(-0.5, min(0.5, f_high))
    h = design_windowed_sinc_bandpass(f_low, f_high, filter_bw)
    if len(h) < 8 * math.log(math.sqrt(len(data))):
        return np.convolve(data, h, "same")
    return fft_convolve_1d(data, h)


# ---- Haar wavelet / modulation detection (Wavelet.py:7-43, AutoInterpretation.py:151-208) -------------------------------
def normalized_haar_wavelet(omega, scale):
    scaled = omega[:] / scale
    scaled[0] = 1.0  # omega[0] == 0: avoid 0/0, the numerator is 0 there anyway
    return (1j * np.square(-1 + np.exp(0.5j * omega))) / scaled


def cwt_haar(x, scale=10):
    num = 2 ** int(np.log2(len(x)))  # truncate to a power of two
    x = x[0:num]
    x_hat = np.fft.fft(x)
    f = 2.0 * np.pi / num
    omega = f * np.concatenate((np.arange(0, num // 2), np.arange(num // 2, num) * -1))
    psi_hat = np.sqrt(2.0 * np.pi * scale) * normalized_haar_wavelet(scale * omega, scale)
    W = np.fft.ifft(x_hat * psi_hat)
    return W[2 * scale: -2 * scale]


def modulation_features(data, wavelet_scale=4, median_filter_order=11):
    """the quantities detect_modulation decides on: (n_nonzero, var_mag, var_norm_mag, var_filtered_mag,
    var_filtered_norm_mag, fsk_test or None) -- None where the reference returns before computing them"""
    n_data = len(data)
    data = data[np.abs(data) > 0]
    if len(data) == 0 or n_data - len(data) > 3:
        return len(data), None
    data = data / np.abs(np.max(data))
    mag = np.abs(cwt_haar(data, scale=wavelet_scale))
    if len(mag) == 0:
        return len(data), None
    norm_mag = np.abs(cwt_haar(data / np.abs(data), scale=wavelet_scale))
    fft = np.fft.fft(data[0: 2 ** int(np.log2(len(data)))])
    fft = np.abs(np.fft.fftshift(fft))
    ten = np.argsort(fft)[::-1][0:10]
    fsk = bool(any(abs(i - ten[0]) >= 10 and fft[i] >= 100 for i in ten))
    return len(data), (float(np.var(mag)), float(np.var(norm_mag)), float(np.var(median_filter(mag, k=median_filter_order))),
                       float(np.var(median_filter(norm_mag, k=median_filter_order))), fsk)


def detect_modulation(data, wavelet_scale=4, median_filter_order=11):
    n_data = len(data)
    nz, feat = modulation_features(data, wavelet_scale, median_filter_order)
    if nz == 0:
        return None
    if n_data - nz > 3:
        return "OOK"
    if feat is None:
        return None
    var_mag, var_norm_mag, var_filtered_mag, var_filtered_norm_mag, fsk = feat
    if all(v < 0.15 for v in (var_mag, var_norm_mag, var_filtered_mag, var_filtered_norm_mag)):
        return "OOK"
    if var_mag > 1.5 * var_norm_mag:
        return "ASK"
    if var_mag > 10 * var_filtered_mag:
        return "PSK"
    return "FSK" if fsk else "OOK"


# ---- capture format conversion (IQArray.py:127-200) ------------------------------------------------------------------
def convert_iq(data, target_dtype):
    """IQArray.convert_to (IQArray.py:127-200) restated with the same numpy operations"""
    _INT_TYPES = (np.uint8, np.int8, np.uint16, np.int16)
    src = data.dtype
    tgt = np.dtype(target_dtype)
    d = data
    if tgt == src:
        return d
    if tgt not in [np.dtype(t) for t in _INT_TYPES + (np.float32,)]:
        raise ValueError("Data type {} not supported".format(target_dtype))
    if src == np.uint8:
        if tgt == np.int8:
            return np.add(d, -128, dtype=np.int8, casting="unsafe")
        if tgt == np.int16:
            return np.add(d, -128, dtype=np.int16, casting="unsafe") << 8
        if tgt == np.uint16:
            return d.astype(np.uint16) << 8
        if tgt == np.float32:
            return np.add(np.multiply(d, 1 / 128, dtype=np.float32), -1.0, dtype=np.float32)
    if src == np.int8:
        if tgt == np.uint8:
            return np.add(d, 128, dtype=np.uint8, casting="unsafe")
        if tgt == np.int16:
            return d.astype(np.int16) << 8
        if tgt == np.uint16:
            return np.add(d, 128, dtype=np.uint16, casting="unsafe") << 8
        if tgt == np.float32:
            return np.multiply(d, 1 / 128, dtype=np.float32)
    if src == np.uint16:
        if tgt == np.int8:
            return (np.add(d, -32768, dtype=np.int16, casting="unsafe") >> 8).astype(np.int8)
        if tgt == np.uint8:
            return (d >> 8).astype(np.uint8)
        if tgt == np.int16:
            return np.add(d, -32768, dtype=np.int16, casting="unsafe")
        if tgt == np.float32:
            return np.add(np.multiply(d, 1 / 32768, dtype=np.float32), -1.0, dtype=np.float32)
    if src == np.int16:
        if tgt == np.int8:
            return (d >> 8).astype(np.int8)
        if tgt == np.uint8:
            return (np.add(d, 32768, dtype=np.uint16, casting="unsafe") >> 8).astype(np.uint8)
        if tgt == np.uint16:
            return np.add(d, 32768, dtype=np.uint16, casting="unsafe")
        if tgt == np.float32:
            return np.multiply(d, 1 / 32768, dtype=np.float32)
    if src == np.float32:
        if tgt == np.int8:
            return np.multiply(d, 127, dtype=np.float32).astype(np.int8)
        if tgt == np.uint8:
            return np.multiply(np.add(d, 1.0, dtype=np.float32), 127, dtype=np.float32).astype(np.uint8)
        if tgt == np.int16:
            return np.multiply(d, 32767, dtype=np.float32).astype(np.int16)
        if tgt == np.uint16:
            return np.multiply(np.add(d, 1.0, dtype=np.float32), 32767, dtype=np.float32).astype(np.uint16)
    raise NotImplementedError("Conversion from {} to {} not supported", src, tgt)


# ---- pulses -> bits (test oracle for bits.cu) ---------------------------------------------------------------------------
def number_to_bits(n: int, length: int) -> list:
    """util.number_to_bits (src/urh/util/util.py): MSB-first bit list of fixed length"""
    return [int(c) for c in format(int(n), "0{}b".format(length))]


def ppseq_to_bits(ppseq, samples_per_symbol, bits_per_symbol, write_bit_sample_pos=True, pause_threshold=8):
    """Sequential restatement of ProtocolAnalyzer._ppseq_to_bits (src/urh/signalprocessing/ProtocolAnalyzer.py:323-414): the
    checker for urh_ppseq_to_bits (bits.cu).  Pinned to the reference's method by tests/test_host_vs_reference.py."""
    import array
    positions, all_positions = array.array("L", []), []
    bits, all_bits = array.array("B", []), []
    pauses = array.array("L", [])
    first, total = 0, 0
    there_was_data = False
    samples_per_bit = int(samples_per_symbol / bits_per_symbol)
    if len(ppseq) > 0 and ppseq[0, 0] == -1:
        first, total = 1, int(ppseq[0, 1])  # capture starts with a pause
    for i in range(first, len(ppseq)):
        kind, num_samples = int(ppseq[i, 0]), int(ppseq[i, 1])
        num_symbols_float = num_samples / samples_per_symbol
        num_symbols = int(num_symbols_float)
        if num_symbols_float - num_symbols > 0.5:
            num_symbols += 1
        if kind == -1:
            if num_symbols <= pause_threshold or pause_threshold == 0:
                bits.extend([0] * (num_symbols * bits_per_symbol))
                if write_bit_sample_pos:
                    positions.extend([total + k * samples_per_bit for k in range(num_symbols * bits_per_symbol)])
            elif not there_was_data:
                bits = array.array("B", [])
                positions = array.array("L", [])
            else:
                if write_bit_sample_pos:
                    positions.append(total)
                    positions.append(total + num_samples)
                    all_positions.append(positions[:])
                    positions = array.array("L", [])
                all_bits.append(bits[:])
                bits = array.array("B", [])
                pauses.append(num_samples)
                there_was_data = False
        else:
            bits.extend(number_to_bits(kind, bits_per_symbol) * num_symbols)
            if not there_was_data and num_symbols > 0:
                there_was_data = True
            if write_bit_sample_pos:
                positions.extend([total + k * samples_per_bit for k in range(num_symbols * bits_per_symbol)])
        total += num_samples
    if there_was_data:
        all_bits.append(bits[:])
        if write_bit_sample_pos:
            all_positions.append(positions[:] + array.array("L", [total]))
        pauses.append(int(ppseq[-1, 1]) if ppseq[-1, 0] == -1 else 0)
    return all_bits, pauses, all_positions


# ---- numpy's float32 pairwise summation, restated (checker for pairwise.cu; pinned to numpy by tests/test_pairwise_model.py) ------
def np_pairwise_sum_f32(a):
    """numpy/_core/src/umath/loops_utils.h.src FLOAT_pairwise_sum on a contiguous float32 array (pure Python: small inputs)"""
    f32 = np.float32
    n = len(a)
    if n < 8:
        r = f32(0.0)
        for x in a:
            r = f32(r + x)
        return r
    if n <= 128:
        r = [a[k] for k in range(8)]
        i = 8
        while i < n - (n % 8):
            for k in range(8):
                r[k] = f32(r[k] + a[i + k])
            i += 8
        res = f32(f32(f32(r[0] + r[1]) + f32(r[2] + r[3])) + f32(f32(r[4] + r[5]) + f32(r[6] + r[7])))
        while i < n:
            res = f32(res + a[i])
            i += 1
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return f32(np_pairwise_sum_f32(a[:n2]) + np_pairwise_sum_f32(a[n2:]))


def np_var_f32(a):
    """np.var of a float32 array as numpy/_core/_methods.py _var computes it: (mean, var), both float32"""
    f32 = np.float32
    a = np.ascontiguousarray(a, dtype=f32)
    n = len(a)
    mean = f32(np.float64(f32(0.0) + np_pairwise_sum_f32(a)) / np.float64(n))
    x = (a - mean).astype(f32)
    x = (x * x).astype(f32)
    return mean, f32(np.float64(f32(0.0) + np_pairwise_sum_f32(x)) / np.float64(n))
