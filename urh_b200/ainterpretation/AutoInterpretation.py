"""Automatic parameter detection on the GPU path (reference: src/urh/ainterpretation/AutoInterpretation.py).

Same module-level functions, arguments and return values as the reference.  The sample-rate work — magnitudes,
chunk statistics, rank-trimmed min/max/variance, histograms, run tables, demodulation — runs in liburh_b200
(stats.cu, digitize.cu); the small data-dependent decisions (which chunks are quiet, which histogram bins are
local maxima, plateau bookkeeping of a few hundred entries per message) stay on the host as in the reference.
Every function accepts host numpy arrays or ``DeviceArray``s.
"""
import ctypes as C
import itertools
import math
from collections import Counter

import numpy as np

from .. import _lib
from ..cythonext import auto_interpretation as c_auto_interpretation
from ..cythonext import signal_functions
from ..cythonext import util
from ..device import DeviceArray, to_device
from . import Wavelet


# ---- small helpers (AutoInterpretation.py:14-57) ----------------------------------------------------------------
def max_without_outliers(data: np.ndarray, z=3):
    if len(data) == 0:
        return None
    return np.max(data[abs(data - np.mean(data)) <= z * np.std(data)])


def min_without_outliers(data: np.ndarray, z=2):
    if len(data) == 0:
        return None
    return np.min(data[abs(data - np.mean(data)) <= z * np.std(data)])


def get_most_frequent_value(values: list):
    """most frequent value; ties resolved towards the LAST of the equally frequent ones in Counter order
    (AutoInterpretation.py:29-47)"""
    if len(values) == 0:
        return None
    ranked = Counter(values).most_common()
    best, top = ranked[0]
    for value, count in ranked:
        if count < top:
            return best
        best = value
    return best


def most_common(values: list):
    """most common value, ties -> first in the list (AutoInterpretation.py:50-57)"""
    counter = Counter(values)
    return max(values, key=counter.get)


# ---- noise level (AutoInterpretation.py:60-91) ------------------------------------------------------------------
def _noise_from_chunk_stats(n, chunksize, sums, maxs, mag_dtype):
    mean_values = (np.asarray(sums, dtype=np.float64) / chunksize).astype(np.float32)
    minimum, maximum = util.minmax(mean_values)
    if maximum == 0 or minimum / maximum > 0.9:
        return 0  # chunk means nearly equal: no noise-only part in the capture
    quiet = np.nonzero(mean_values <= 1.1 * np.min(mean_values))[0]
    if len(quiet) == 0:
        return 0
    result = np.max(np.asarray(maxs)[quiet].astype(mag_dtype))
    return math.ceil(result * 10000) / 10000


def _chunking(n):
    chunksize = max(1, int(n * 1 / 100))
    return chunksize, n // chunksize


def detect_noise_level(magnitudes):
    """`magnitudes`: float32/float64 array (host or device)."""
    n = len(magnitudes)
    if n <= 3:
        return 0
    on_device = isinstance(magnitudes, DeviceArray)
    if not on_device:
        magnitudes = np.ascontiguousarray(magnitudes)
        if magnitudes.dtype not in (np.float32, np.float64):
            magnitudes = magnitudes.astype(np.float64)
    ctx = magnitudes.ctx if on_device else _lib.default_context()
    d = magnitudes if on_device else to_device(magnitudes, ctx)
    chunksize, nchunks = _chunking(n)
    sums = np.empty(nchunks, dtype=np.float64)
    maxs = np.empty(nchunks, dtype=np.float64)
    ctx.check(ctx.lib.urh_noise_chunk_stats(ctx.handle, C.c_void_p(d.ptr), int(d.dtype == np.float64), n, chunksize, nchunks,
                                            sums.ctypes.data_as(C.c_void_p), maxs.ctypes.data_as(C.c_void_p)))
    return _noise_from_chunk_stats(n, chunksize, sums, maxs, d.dtype)


def noise_level_streams(n: int, dtype, budget: int) -> bool:
    """whether detect_noise_level_iq streams a host capture of n samples: its resident call (the capture uploaded whole) does not
    fit the device budget (signal_functions.filter_use_stream's rule)"""
    if n <= 3:
        return False
    chunksize, nchunks = _chunking(n)
    return signal_functions.filter_use_stream(_lib.FILTER_NOISE, n, 0, dtype, chunksize, nchunks, budget)


def detect_noise_level_iq(iq):
    """detect_noise_level(IQArray(iq).magnitudes) without materialising the float64 magnitude array
    (8 B/sample in the reference, SURVEY §5): `iq` is an (n,2) array (host or device).  A host capture whose upload does not fit
    the device budget streams through the device (urh_noise_chunk_stats_iq_stream; the same sums and maxima)."""
    n = len(iq)
    if n <= 3:
        return 0
    on_device = isinstance(iq, DeviceArray)
    ctx = iq.ctx if on_device else _lib.default_context()
    chunksize, nchunks = _chunking(n)
    sums = np.empty(nchunks, dtype=np.float64)
    maxs = np.empty(nchunks, dtype=np.float64)
    if not on_device:
        iq = np.ascontiguousarray(iq)
        if noise_level_streams(n, iq.dtype, signal_functions.device_budget(ctx)):
            ctx.check(ctx.lib.urh_noise_chunk_stats_iq_stream(ctx.handle, iq.ctypes.data_as(C.c_void_p), _lib.dtype_code(iq.dtype), n,
                                                              chunksize, nchunks, signal_functions.FILTER_STREAM_CHUNK,
                                                              signal_functions.STREAM_RING, sums.ctypes.data_as(C.c_void_p),
                                                              maxs.ctypes.data_as(C.c_void_p)))
            return _noise_from_chunk_stats(n, chunksize, sums, maxs, np.float64)
    d = iq if on_device else to_device(iq, ctx)
    ctx.check(ctx.lib.urh_noise_chunk_stats_iq(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(d.dtype), n, chunksize, nchunks,
                                               sums.ctypes.data_as(C.c_void_p), maxs.ctypes.data_as(C.c_void_p)))
    return _noise_from_chunk_stats(n, chunksize, sums, maxs, np.float64)


# ---- segmentation (AutoInterpretation.py:94-148) -----------------------------------------------------------------
def segment_messages_from_magnitudes(magnitudes, noise_threshold: float):
    return c_auto_interpretation.segment_messages_from_magnitudes(magnitudes, noise_threshold)


def segment_messages_iq(iq, noise_threshold: float) -> list:
    """segment_messages_from_magnitudes(get_magnitudes(iq), noise_threshold) of an (n,2) capture (host or device): the float64
    magnitudes estimate() segments.  A host capture whose resident call (capture, magnitudes, run tables) does not fit the device
    budget streams through the device chunk by chunk (urh_segment_messages_iq_stream; the same segments)."""
    n = len(iq)
    if n == 0:
        return []
    on_device = isinstance(iq, DeviceArray)
    ctx = iq.ctx if on_device else _lib.default_context()
    if not on_device:
        iq = np.ascontiguousarray(iq)
        if signal_functions.use_stream(n, iq.dtype, 0, _lib.STREAM_SEGMENT_MESSAGES, signal_functions.device_budget(ctx)):
            k = C.c_int64(0)
            ctx.check(ctx.lib.urh_segment_messages_iq_stream(ctx.handle, iq.ctypes.data_as(C.c_void_p), _lib.dtype_code(iq.dtype), n,
                                                             float(noise_threshold), signal_functions.STREAM_CHUNK,
                                                             signal_functions.STREAM_RING, C.byref(k)))
            seg = np.empty((k.value, 2), dtype=np.int64)
            ctx.check(ctx.lib.urh_fetch_segments(ctx.handle, seg.ctypes.data_as(C.c_void_p), k.value))
            return [(int(a), int(b)) for a, b in seg]
    d_iq = iq if on_device else to_device(iq, ctx)
    d_mag = util.get_magnitudes(d_iq)
    try:
        return segment_messages_from_magnitudes(d_mag, noise_threshold)
    finally:
        d_mag.free()


def merge_message_segments_for_ook(segments: list):
    if len(segments) <= 1:
        return segments
    starts = np.array([s for s, _ in segments], dtype=np.int64)
    ends = np.array([e for _, e in segments], dtype=np.int64)
    pauses = (starts[1:] - ends[:-1]).astype(np.uint64)
    pulses = (ends - starts).astype(np.uint64)
    min_pulse_length = min_without_outliers(pulses, z=1)
    large = np.nonzero(pauses >= 8 * min_pulse_length)[0]
    result = []
    bounds = [0] + [int(i) + 1 for i in large] + [len(segments)]
    for a, b in zip(bounds[:-1], bounds[1:]):
        begin = segments[a][0]
        length = sum(segments[j][1] - segments[j][0] for j in range(a, b))
        length += sum(segments[j][0] - segments[j - 1][1] for j in range(a + 1, b))
        result.append((begin, begin + length))
    return result


# ---- modulation detection (AutoInterpretation.py:151-223) --------------------------------------------------------
def modulation_features(data, wavelet_scale=4, median_filter_order=11):
    """The sample-rate part of detect_modulation on the GPU (modulation.cu): -> (feat[8], spec[23]), see urh_b200.h."""
    on_device = isinstance(data, DeviceArray)
    if on_device:
        ctx, d = data.ctx, data
        if data.dtype != np.complex64:
            raise ValueError("complex64 message expected")
    else:
        data = np.ascontiguousarray(data, dtype=np.complex64)
        ctx = _lib.default_context()
        d = to_device(data.view(np.float32), ctx) if len(data) else None
    feat, spec = np.zeros(8), np.full(23, -1.0)
    if len(data):
        ctx.check(ctx.lib.urh_modulation_features(ctx.handle, C.c_void_p(d.ptr), len(data), int(wavelet_scale), int(median_filter_order),
                                                  feat.ctypes.data_as(C.c_void_p), spec.ctypes.data_as(C.c_void_p)))
    return feat, spec


def _fsk_peak_test(spec) -> bool:
    """`any(abs(i - top) >= 10 and fft[i] >= 100 for i in ten_greatest)` from the device's spectrum features: the largest
    value >= 10 bins from the arg-max is one of the ten greatest iff fewer than ten bins (all of them within 9 bins of the
    arg-max) exceed it; every other far bin among the ten greatest is smaller still."""
    far_index, far_value = int(spec[2]), spec[3]
    if far_index < 0 or far_value < 100:
        return False
    return int(np.sum(spec[4:23] > far_value)) < 10


def detect_modulation(data, wavelet_scale=4, median_filter_order=11) -> str:
    """AutoInterpretation.py:151-208; the decision thresholds are the reference's, the features come from the GPU."""
    n_data = len(data)
    feat, spec = modulation_features(data, wavelet_scale, median_filter_order)
    n_nonzero = int(feat[0])
    if n_nonzero == 0:
        return None
    if n_data - n_nonzero > 3:
        return "OOK"
    if int(feat[2]) == 0:
        return None  # message shorter than the wavelet's support
    var_mag, var_norm_mag, var_filtered_mag, var_filtered_norm_mag = feat[3:7]
    if all(v < 0.15 for v in (var_mag, var_norm_mag, var_filtered_mag, var_filtered_norm_mag)):
        return "OOK"
    if var_mag > 1.5 * var_norm_mag:
        return "ASK"
    if var_mag > 10 * var_filtered_mag:
        return "PSK"
    # FSK has at least two spectral peaks, a lone OOK pulse has one
    return "FSK" if _fsk_peak_test(spec) else "OOK"


def detect_modulation_for_messages(signal, message_indices: list) -> str:
    """each message converted from its own slice: the same complex64 values as slicing the whole capture's conversion (the
    conversion is element-wise), without converting or uploading the rest of the capture"""
    max_messages = 100
    found = []
    for start, end in message_indices[0:max_messages]:
        mod = detect_modulation(signal.subarray(start, end).as_complex64())
        if mod is not None:
            found.append(mod)
    if len(found) == 0:
        return None
    return most_common(found)


# ---- center detection (AutoInterpretation.py:226-277) --------------------------------------------------------------
def detect_center(rectangular_signal, max_size=None):
    """Histogram peak pair of the demodulated signal.  Sample-rate part on the GPU: rank trimming of the
    non-noise samples, min/max/variance, histogram; peak picking (a few thousand bins) on the host.
    np.var's float32 pairwise sums are replayed bit for bit on the device (pairwise.cu), so bin edges, histogram and center
    are bit-identical to the reference's."""
    on_device = isinstance(rectangular_signal, DeviceArray)
    n = len(rectangular_signal)
    if n == 0:
        return None
    ctx = rectangular_signal.ctx if on_device else _lib.default_context()
    d = rectangular_signal if on_device else to_device(np.ascontiguousarray(rectangular_signal, dtype=np.float32), ctx)
    st = np.zeros(7, dtype=np.float64)
    ctx.check(ctx.lib.urh_center_stats(ctx.handle, C.c_void_p(d.ptr), n, -1 if max_size is None else int(max_size),
                                       st.ctypes.data_as(C.c_void_p)))
    return _center_from_stats(ctx, d, n, st, ctx.lib.urh_center_histogram)


def center_bin_edges(st):
    """detect_center's bin edges (AutoInterpretation.py:206-211): np.arange(min, max + var, var) of the trimmed window;
    None when the window is empty or constant."""
    r0, r1 = int(st[1]), int(st[2])
    if r1 <= r0:
        return None
    hist_min, hist_max = float(st[3]), float(st[4])
    hist_step = float(np.float32(st[6]))
    try:
        with np.errstate(all="ignore"):
            edges = np.arange(hist_min, hist_max + hist_step, hist_step)
        if len(edges) < 2:
            raise ValueError("need at least two bin edges")
    except (ZeroDivisionError, ValueError):
        return None  # constant segment: no center
    return edges


def pick_center_from_histogram(y, edges):
    """Peak picking of detect_center (AutoInterpretation.py:213-240): the two most populated bins that dominate their
    5 % neighbourhood; center = mean of their left edges."""
    nbins = len(edges) - 1
    window = max(2, int(0.05 * nbins) + 1)
    # same decision as the reference's loop, evaluated for every bin at once: a peak exceeds every neighbour within
    # `window` bins on both sides (bins beyond the ends count as 0)
    y = np.asarray(y)
    padded = np.concatenate([np.zeros(window, dtype=y.dtype), y, np.zeros(window, dtype=y.dtype)])
    is_peak = np.ones(nbins, dtype=bool)
    for i in range(1, window):
        is_peak &= (y > padded[window + i:window + i + nbins]) & (y > padded[window - i:window - i + nbins])
    levels = []
    for index in np.argsort(y)[::-1]:
        if is_peak[index]:
            levels.append(edges[index])
            if len(levels) == 2:
                break
    if len(levels) == 0:
        return None
    return np.mean(levels)


def _center_from_stats(ctx, d, n, st, histogram_entry):
    """Host half of detect_center: bin edges from the trimmed min/max/variance, the device histogram, peak picking."""
    edges = center_bin_edges(st)
    if edges is None:
        return None
    r0, r1 = int(st[1]), int(st[2])
    nbins = len(edges) - 1
    y = np.zeros(nbins, dtype=np.int64)
    # np.arange fills start + i*delta with delta = (start + step) - start
    ctx.check(histogram_entry(ctx.handle, C.c_void_p(d.ptr), n, r0, r1, C.c_double(edges[0]),
                              C.c_double(edges[1] - edges[0]), nbins, y.ctypes.data_as(C.c_void_p)))
    return pick_center_from_histogram(y, edges)


def demod_detect_center(iq, noise_mag: float, mod_type: str, max_size=None, out=None, bitwise=False):
    """afp_demod (ASK/FSK) + detect_center sharing ONE pass over the IQ samples: the demodulator leaves per-tile
    {count, min, max, sum, sumsq} of the kept samples, so detect_center only adds its histogram pass over qad.
    Returns (qad DeviceArray, center or None); same values as afp_demod followed by detect_center.
    ``out``: optional float32[n] DeviceArray to receive qad."""
    from urh_b200.cythonext.signal_functions import _check_iq
    iq = _check_iq(iq)
    on_device = isinstance(iq, DeviceArray)
    ctx = iq.ctx if on_device else _lib.default_context()
    n = len(iq)
    code = _lib.demod_mod_code(mod_type)
    if code not in (_lib.MOD_ASK, _lib.MOD_FSK) or n <= 2:
        raise ValueError("demod_detect_center handles ASK and FSK captures of more than 2 samples")
    d_iq = iq if on_device else to_device(iq, ctx)
    if out is not None and (not isinstance(out, DeviceArray) or out.dtype != np.float32 or out.shape != (n,)):
        raise ValueError("out must be a float32 DeviceArray of n samples")
    qad = out if out is not None else DeviceArray(ctx, (n,), np.float32)
    kept = C.c_int64(0)
    ctx.check(ctx.lib.urh_afp_demod_tiles(ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(d_iq.dtype), n, float(noise_mag),
                                          code, C.c_void_p(qad.ptr), 0, C.byref(kept)))
    st = fused_window_stats(ctx, qad, n, kept.value, max_size, bitwise)
    return qad, _center_from_stats(ctx, qad, n, st, ctx.lib.urh_center_histogram_tiles)


# The fused steps take np.var(rect) from the demodulator's double tile sums, (Σx² - n·mean²) / n.  numpy's float32 variance of
# the same window differs from that by about the square of its float32 mean's error, which is up to ~2^-19 of |mean| (pairwise
# sums, n up to 2^30).  Below var = mean² · 2^-14 (a strong, nearly constant level) that difference outgrows the variance's own
# float32 rounding and moves the bin width, so there the steps replay numpy's variance instead (k_center_plan: state 2).
FUSED_VAR_MIN_RATIO = 2.0 ** -14


def fused_variance_stands(st):
    """whether the double tile-sum variance in st (center_stats_from_window) may stand in for numpy's float32 np.var"""
    return bool(st[6] >= st[5] * st[5] * FUSED_VAR_MIN_RATIO)


def fused_window_stats(ctx, qad, n, kept, max_size=None, bitwise=False):
    """detect_center's window statistics of qad from the tile table in the arena: the double tile-sum variance, or numpy's float32
    variance replayed bit for bit (pairwise.cu) with ``bitwise`` or where the double one may not stand in for it"""
    r0, r1 = center_rank_window(kept, max_size)
    w = np.zeros(5, dtype=np.float64)
    ctx.check(ctx.lib.urh_center_window_stats(ctx.handle, C.c_void_p(qad.ptr), n, r0, r1, w.ctypes.data_as(C.c_void_p)))
    st = center_stats_from_window(kept, r0, r1, w)
    if int(st[2]) > int(st[1]) and (bitwise or not fused_variance_stands(st)):
        # np.var(rect) as numpy computes it (float32 pairwise sums replayed on the device): two more passes over the window,
        # and the center is bit-identical to the reference's instead of agreeing to ~1e-6
        mv = np.zeros(2, dtype=np.float64)
        ctx.check(ctx.lib.urh_center_window_var(ctx.handle, C.c_void_p(qad.ptr), n, r0, r1, mv.ctypes.data_as(C.c_void_p)))
        st[5], st[6] = mv[0], mv[1]
    return st


def center_rank_window(kept: int, max_size=None):
    """detect_center's trimming (AutoInterpretation.py:196-200): ranks [5 %, 95 %) of the kept samples, capped by max_size."""
    r0, r1 = int(0.05 * kept), int(0.95 * kept)
    if max_size is not None and r1 - r0 > int(max_size):
        r1 = r0 + int(max_size)
    return r0, r1


def center_stats_from_window(kept, r0, r1, w):
    """{count, min, max, sum, sumsq} of the window -> the 7-slot layout urh_center_stats returns."""
    st = np.zeros(7, dtype=np.float64)
    st[0], st[1], st[2] = kept, r0, r1
    cnt = int(w[0])
    if cnt <= 0:
        st[2] = st[1]  # empty window: no center
        return st
    mean = w[3] / cnt
    ss = max(0.0, w[4] - cnt * mean * mean)
    st[3], st[4], st[5], st[6] = w[1], w[2], mean, ss / cnt
    return st


# ---- plateau bookkeeping (AutoInterpretation.py:280-370) ---------------------------------------------------------------
def estimate_tolerance_from_plateau_lengths(plateau_lengths, relative_max=0.05) -> int:
    if len(plateau_lengths) <= 1:
        return None
    unique = np.unique(plateau_lengths)
    limit = relative_max * max_without_outliers(unique, z=2)
    if unique[0] > 1 and unique[0] >= limit:
        return 0
    result = 0
    for value in unique:
        if value > 1 and value >= limit:
            break
        result = value
    return result


def merge_plateau_lengths(plateau_lengths, tolerance=None) -> list:
    if tolerance is None:
        tolerance = estimate_tolerance_from_plateau_lengths(plateau_lengths)
    if tolerance == 0 or tolerance is None:
        return plateau_lengths
    return c_auto_interpretation.merge_plateaus(plateau_lengths, tolerance, max_count=10000)


def round_plateau_lengths(plateau_lengths: list):
    """round in place to the digit count of the median length (99 -> 100, 293 -> 300)"""
    digit_counts = [len(str(p)) for p in plateau_lengths]
    n_digits = min(3, int(np.percentile(digit_counts, 50)))
    f = 10 ** (n_digits - 1)
    for i, plateau_len in enumerate(plateau_lengths):
        plateau_lengths[i] = int(round(plateau_len / f)) * f


def get_tolerant_greatest_common_divisor(numbers):
    gcds = [math.gcd(x, y) for x, y in itertools.combinations(numbers, 2) if math.gcd(x, y) != 1]
    if len(gcds) == 0:
        return 1
    return get_most_frequent_value(gcds)


def get_bit_length_from_plateau_lengths(merged_plateau_lengths) -> int:
    if len(merged_plateau_lengths) == 0:
        return 0
    if len(merged_plateau_lengths) == 1:
        return int(merged_plateau_lengths[0])
    round_plateau_lengths(merged_plateau_lengths)
    histogram = c_auto_interpretation.get_threshold_divisor_histogram(merged_plateau_lengths)
    if len(histogram) == 0:
        return 0
    order = np.argsort(histogram)[::-1]
    max_count = histogram[order[0]]
    result = order[0]
    for i in range(1, len(order)):
        if histogram[order[i]] < 0.25 * max_count:
            break
        if order[i] <= 0.5 * result:
            result = order[i]
    return int(result)


# ---- orchestrator (AutoInterpretation.py:373-471) ------------------------------------------------------------------------
def estimate_streams(n: int, dtype, budget: int) -> bool:
    """whether estimate() takes its host path: the resident path's footprint (urh_stream_footprint, URH_STREAM_ENTRY_ESTIMATE:
    capture, float64 magnitudes, the resident order-2 PSK demodulation, the largest of the three) exceeds the device budget"""
    return signal_functions.stream_footprint(n, dtype, 0, _lib.STREAM_ESTIMATE | _lib.STREAM_RESIDENT) > budget


def _demodulate(iq, noise, modulation):
    if modulation in ("OOK", "ASK"):
        return signal_functions.afp_demod(iq, noise, "ASK", 2)
    if modulation in ("FSK", "PSK"):
        return signal_functions.afp_demod(iq, noise, modulation, 2)
    raise ValueError("Unsupported Modulation")


def _center_and_plateaus(msg):
    center = detect_center(msg)
    if center is None:
        return None, None
    return center, c_auto_interpretation.get_plateau_lengths(msg, center, percentage=25)


def estimate(iq_array, noise: float = None, modulation: str = None) -> dict:
    """AutoInterpretation.py:373-471.  A capture whose resident path does not fit the device budget (estimate_streams) stays on the
    host: the noise level and the segmentation stream through the device, afp_demod streams (ASK / FSK / PSK), and each message's
    demodulated slice is uploaded once for its center and plateau lengths.  Both paths give the same dict.  Limit: a single message
    whose per-message work does not fit the device raises MemoryError."""
    from ..signalprocessing.IQArray import IQArray

    if isinstance(iq_array, np.ndarray):
        iq_array = IQArray(iq_array)
    ctx = _lib.default_context()
    host = np.ascontiguousarray(iq_array._peek())
    on_host = estimate_streams(len(host), host.dtype, signal_functions.device_budget(ctx))
    if on_host:
        noise = detect_noise_level_iq(host) if noise is None else noise
        message_indices = segment_messages_iq(host, noise)
    else:
        d_iq = to_device(host, ctx)  # one upload, everything below stays in HBM
        d_mag = util.get_magnitudes(d_iq)
        noise = detect_noise_level(d_mag) if noise is None else noise
        message_indices = segment_messages_from_magnitudes(d_mag, noise_threshold=noise)
        d_mag.free()
    modulation = detect_modulation_for_messages(iq_array, message_indices) if modulation is None else modulation
    if modulation is None:
        return None
    if modulation == "OOK":
        message_indices = merge_message_segments_for_ook(message_indices)
    data = _demodulate(host if on_host else d_iq, noise, modulation)

    centers, bit_lengths, tolerances = [], [], []
    for start, end in message_indices:
        msg = data[int(start):int(end)]
        if on_host:   # the message's qad uploaded once (freed with the DeviceArray)
            try:
                center, plateau_lengths = _center_and_plateaus(to_device(np.ascontiguousarray(msg), ctx))
            except MemoryError as e:
                raise MemoryError("estimate: the message [%d, %d) of %d samples does not fit the device" % (start, end, end - start)) from e
        else:
            center, plateau_lengths = _center_and_plateaus(msg)
        if center is None:
            continue
        tolerance = estimate_tolerance_from_plateau_lengths(plateau_lengths)
        if tolerance is None:
            tolerance = 0
        else:
            tolerances.append(tolerance)
        merged_lengths = merge_plateau_lengths(plateau_lengths, tolerance=tolerance)
        if len(merged_lengths) < 2:
            continue
        bit_length = get_bit_length_from_plateau_lengths(merged_lengths)
        if bit_length > tolerance + 1:
            centers.append(center)
            bit_lengths.append(bit_length)

    if modulation == "OOK" or modulation == "ASK":
        center = min_without_outliers(np.array(centers), z=2)
        if center is None:
            return None
    elif len(centers) > 0:
        center = np.mean(centers)
    else:
        return None
    bit_length = get_most_frequent_value(bit_lengths)
    if bit_length is None:
        return None
    try:
        tolerance = np.percentile(tolerances, 50)
    except IndexError:
        tolerance = max(1, int(0.05 * bit_length))
    return {
        "modulation_type": "ASK" if modulation == "OOK" else modulation,
        "bit_length": bit_length,
        "center": center,
        "tolerance": int(tolerance),
        "noise": noise,
    }
