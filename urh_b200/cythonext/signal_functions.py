"""CUDA drop-in for ``urh.cythonext.signal_functions`` (reference: src/urh/cythonext/signal_functions.pyx)."""
import ctypes as C
import os

import numpy as np

from .. import _lib
from ..device import DeviceArray, to_device

_IQ_DTYPES = (np.int8, np.uint8, np.int16, np.uint16, np.float32)


def _check_iq(samples):
    """Mimic the Cython fused-type dispatch of ``IQ samples`` (util.pxd:1-10)."""
    if isinstance(samples, DeviceArray):
        if samples.ndim != 2 or samples.shape[1] != 2:
            raise ValueError("Buffer has wrong number of dimensions (expected 2)")
        if samples.dtype not in [np.dtype(t) for t in _IQ_DTYPES]:
            raise TypeError("No matching signature found")
        return samples
    samples = np.asarray(samples) if not isinstance(samples, np.ndarray) else samples
    if samples.ndim != 2:
        raise TypeError("No matching signature found")
    if samples.dtype not in [np.dtype(t) for t in _IQ_DTYPES]:
        raise TypeError("No matching signature found")
    if samples.shape[1] != 2 and len(samples):
        raise ValueError("IQ samples must have shape (n, 2)")
    if not samples.flags.c_contiguous:
        raise ValueError("ndarray is not C-contiguous")
    return samples


# ---- captures larger than device memory -------------------------------------------------------------------------------
# A host capture whose resident footprint exceeds the device budget goes through a ring of STREAM_RING device slots of
# STREAM_CHUNK samples (urh_*_stream, DESIGN.md §4.11); the results are bit-identical.  Pinned host memory (PinnedArray) lets the
# copies overlap the kernels; a pageable array or np.memmap works too, but then every copy blocks the calling thread.
STREAM_CHUNK = 1 << 24
STREAM_RING = 2
# PSK streams in longer chunks: the speculative Costas loop (DESIGN.md §4.3) sizes its own sub-chunks from the length it is given, and
# a short ring chunk forces short sub-chunks whose warm-up outweighs them.  Chosen by measurement (DESIGN.md §4.11).
PSK_STREAM_CHUNK = 1 << 26


def psk_entry(mod_order: int) -> int:
    """urh_stream_footprint flags of a PSK call with Costas loop order mod_order (orders above 4 run as 4)"""
    return _lib.STREAM_PSK | (_lib.STREAM_PSK4 if int(mod_order) >= 4 else 0)


def stream_footprint(n: int, dtype, tolerance: int, entry: int, chunk_samples: int = STREAM_CHUNK, ring: int = STREAM_RING,
                     rows: int = -1) -> int:
    """device bytes a streamed call (or, with _lib.STREAM_RESIDENT in entry, the resident call) needs; no device involved.
    rows: pulse-table rows to budget for (-1: the bound no capture exceeds, -2: the resident call's up-front reservation)"""
    out = C.c_int64(0)
    rc = _lib.load_library().urh_stream_footprint(int(n), _lib.dtype_code(dtype) if dtype is not None else _lib.DT_F32, int(tolerance),
                                                  int(chunk_samples), int(ring), int(entry), int(rows), C.byref(out))
    if rc != _lib.URH_OK:
        raise ValueError("urh_stream_footprint: invalid arguments")
    return out.value


def device_budget(ctx) -> int:
    """free device memory less a margin; $URH_B200_DEVICE_BUDGET (bytes, read per call) lowers it"""
    free, total = C.c_size_t(0), C.c_size_t(0)
    ctx.check(ctx.lib.urh_mem_get_info(ctx.handle, C.byref(free), C.byref(total)))
    budget = free.value - max(1 << 29, total.value // 32)
    env = os.environ.get("URH_B200_DEVICE_BUDGET")
    if env:
        budget = min(budget, int(env))
    return budget


def use_stream(n: int, dtype, tolerance: int, entry: int, budget: int) -> bool:
    """stream when the resident call's footprint (with the pulse rows it reserves up front, rows = -2) exceeds the budget"""
    return stream_footprint(n, dtype, tolerance, entry | _lib.STREAM_RESIDENT, rows=-2) > budget


# The band-pass, FIR and DC filters and the spectrogram stream through the windowed ring (urh_*_stream of filter.cu and spectrogram.cu,
# DESIGN.md §4.11) on the same rule: a host input whose resident call does not fit the device budget.
FILTER_STREAM_CHUNK = 1 << 24


def filter_footprint(entry: int, n: int, out_len: int, dtype, p0: int, p1: int, chunk_samples: int = FILTER_STREAM_CHUNK,
                     ring: int = STREAM_RING, resident: bool = False, cmap_entries: int = 0) -> int:
    """device bytes of a streamed filter / spectrogram call (entry = _lib.FILTER_*; p0, p1 = taps and offset, or W and hop;
    cmap_entries: the colormap's entries, images only), or of its resident call fed from the host with resident=True; no device
    involved (urh_stream_filter_footprint)"""
    out = C.c_int64(0)
    rc = _lib.load_library().urh_stream_filter_footprint(int(entry), int(n), int(out_len), _lib.dtype_code(dtype), int(p0), int(p1),
                                                         int(cmap_entries), int(chunk_samples), int(ring), int(bool(resident)),
                                                         C.byref(out))
    if rc != _lib.URH_OK:
        raise ValueError("urh_stream_filter_footprint: invalid arguments")
    return out.value


def filter_use_stream(entry: int, n: int, out_len: int, dtype, p0: int, p1: int, budget: int, cmap_entries: int = 0) -> bool:
    """stream when the resident call's footprint exceeds the budget (use_stream's rule)"""
    return filter_footprint(entry, n, out_len, dtype, p0, p1, resident=True, cmap_entries=cmap_entries) > budget


def _host_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def afp_demod(samples, noise_mag: float, mod_type: str, mod_order: int, costas_loop_bandwidth: float = 0.1):
    """signal_functions.pyx:333-378.  Returns float32[n] (numpy for numpy input, DeviceArray for device input)."""
    samples = _check_iq(samples)
    on_device = isinstance(samples, DeviceArray)
    ctx = samples.ctx if on_device else _lib.default_context()
    n = len(samples)
    if n == 0:
        return DeviceArray(ctx, (0,), np.float32) if on_device else np.zeros(0, dtype=np.float32)
    code = _lib.demod_mod_code(mod_type)
    if (not on_device and n > 2 and code in (_lib.MOD_ASK, _lib.MOD_FSK)
            and use_stream(n, samples.dtype, 0, _lib.STREAM_AFP_DEMOD, device_budget(ctx))):
        host = np.empty(n, dtype=np.float32)
        ctx.check(ctx.lib.urh_afp_demod_stream(ctx.handle, _host_ptr(samples), _lib.dtype_code(samples.dtype), n, float(noise_mag), code,
                                               STREAM_CHUNK, STREAM_RING, _host_ptr(host)))
        return host
    if (not on_device and n > 2 and code == _lib.MOD_PSK
            and use_stream(n, samples.dtype, 0, _lib.STREAM_AFP_DEMOD | psk_entry(mod_order), device_budget(ctx))):
        host = np.empty(n, dtype=np.float32)
        ctx.check(ctx.lib.urh_afp_demod_psk_stream(ctx.handle, _host_ptr(samples), _lib.dtype_code(samples.dtype), n, float(noise_mag),
                                                   int(mod_order), float(costas_loop_bandwidth), PSK_STREAM_CHUNK, STREAM_RING,
                                                   _host_ptr(host)))
        return host
    d_iq = samples if on_device else to_device(samples, ctx)
    out = DeviceArray(ctx, (n,), np.float32)
    ctx.check(
        ctx.lib.urh_afp_demod(
            ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(d_iq.dtype), n, float(noise_mag), code if code >= 0 else 99,
            int(mod_order), float(costas_loop_bandwidth), C.c_void_p(out.ptr),
        )
    )
    return out if on_device else out.get()


def get_center_thresholds(center: float, spacing: float, modulation_order: int) -> np.ndarray:
    """signal_functions.pyx:380-390 (host arithmetic; float32)."""
    lib = _lib.load_library()
    out = np.empty(max(int(modulation_order) - 1, 0), dtype=np.float32)
    if len(out):
        lib.urh_get_center_thresholds(float(center), float(spacing), int(modulation_order), out.ctypes.data_as(C.c_void_p))
    return out


def _fetch_pulses(ctx, k: int, out=None) -> np.ndarray:
    """the pulse table of the last digitizer call; ``out``: a caller-owned int64 buffer with room for k rows (pinned memory
    makes the download a true DMA: PinnedArray((rows, 2), np.int64).array) — a view of its first k rows is returned"""
    if out is not None and out.dtype == np.int64 and out.size >= 2 * k and out.flags.c_contiguous:
        rows = out.reshape(-1)[: 2 * k].reshape(k, 2)
    else:
        rows = np.empty((k, 2), dtype=np.int64)
    if k:
        ctx.check(ctx.lib.urh_fetch_pulses(ctx.handle, rows.ctypes.data_as(C.c_void_p), k))
    return rows


def grab_pulse_lens(samples, center: float, tolerance: int, modulation_type: str, samples_per_symbol: int,
                    bits_per_symbol: int = 1, center_spacing: float = 0.1) -> np.ndarray:
    """signal_functions.pyx:392-495.  ``samples`` float32[n] (numpy or DeviceArray) -> int64[k,2] (numpy)."""
    on_device = isinstance(samples, DeviceArray)
    if not on_device:
        if not isinstance(samples, np.ndarray) or samples.dtype != np.float32 or samples.ndim != 1:
            raise ValueError("Buffer dtype mismatch, expected 'float' (1-D float32)")
        if not samples.flags.c_contiguous:
            raise ValueError("ndarray is not C-contiguous")
    elif samples.dtype != np.float32 or samples.ndim != 1:
        raise ValueError("Buffer dtype mismatch, expected 'float' (1-D float32)")
    if not 0 <= int(tolerance) <= 0xFFFF:
        raise OverflowError("value too large to convert to uint16_t")
    if not 0 <= int(bits_per_symbol) <= 0xFF:
        raise OverflowError("value too large to convert to uint8_t")
    ctx = samples.ctx if on_device else _lib.default_context()
    n = len(samples)
    if n == 0:
        return np.zeros((0, 2), dtype=np.int64)
    k = C.c_int64(0)
    code = _lib.demod_mod_code(modulation_type)
    if not on_device and use_stream(n, None, tolerance, _lib.STREAM_GRAB_PULSE_LENS, device_budget(ctx)):
        ctx.check(ctx.lib.urh_grab_pulse_lens_stream(ctx.handle, _host_ptr(samples), 0, n, float(center), int(tolerance),
                                                     code if code >= 0 else 99, int(samples_per_symbol), int(bits_per_symbol),
                                                     float(center_spacing), STREAM_CHUNK, STREAM_RING, C.byref(k)))
        return _fetch_pulses(ctx, k.value)
    d = samples if on_device else to_device(samples, ctx)
    ctx.check(
        ctx.lib.urh_grab_pulse_lens(
            ctx.handle, C.c_void_p(d.ptr), n, float(center), int(tolerance), code if code >= 0 else 99,
            int(samples_per_symbol), int(bits_per_symbol), float(center_spacing), C.byref(k),
        )
    )
    return _fetch_pulses(ctx, k.value)


def demod_digitize(samples, noise_mag: float, mod_type: str, center: float, tolerance: int, samples_per_symbol: int,
                   bits_per_symbol: int = 1, center_spacing: float = 0.1, return_qad: bool = True):
    """Fused afp_demod + grab_pulse_lens in ONE pass over the IQ samples (addition to the reference API; same results as
    calling the two reference functions back to back).  Returns (qad or None, int64[k,2])."""
    samples = _check_iq(samples)
    on_device = isinstance(samples, DeviceArray)
    ctx = samples.ctx if on_device else _lib.default_context()
    n = len(samples)
    if n == 0:
        return (np.zeros(0, np.float32) if return_qad else None), np.zeros((0, 2), dtype=np.int64)
    k = C.c_int64(0)
    code = _lib.demod_mod_code(mod_type)
    entry = _lib.STREAM_DEMOD_DIGITIZE | (_lib.STREAM_QAD_OUT if return_qad else 0)
    if (not on_device and n > 2 and code in (_lib.MOD_ASK, _lib.MOD_FSK)
            and use_stream(n, samples.dtype, tolerance, entry, device_budget(ctx))):
        host = np.empty(n, dtype=np.float32) if return_qad else None
        ctx.check(ctx.lib.urh_demod_digitize_stream(ctx.handle, _host_ptr(samples), _lib.dtype_code(samples.dtype), n, float(noise_mag), code,
                                                    float(center), int(tolerance), int(samples_per_symbol), int(bits_per_symbol),
                                                    float(center_spacing), STREAM_CHUNK, STREAM_RING,
                                                    _host_ptr(host) if host is not None else None, C.byref(k)))
        return host, _fetch_pulses(ctx, k.value)
    # PSK: the Costas loop of order 2^bits_per_symbol, as the resident call runs it
    if (not on_device and n > 2 and code == _lib.MOD_PSK
            and use_stream(n, samples.dtype, tolerance, entry | psk_entry(1 << int(bits_per_symbol)), device_budget(ctx))):
        host = np.empty(n, dtype=np.float32) if return_qad else None
        ctx.check(ctx.lib.urh_demod_digitize_psk_stream(ctx.handle, _host_ptr(samples), _lib.dtype_code(samples.dtype), n, float(noise_mag),
                                                        float(center), int(tolerance), int(samples_per_symbol), int(bits_per_symbol),
                                                        float(center_spacing), PSK_STREAM_CHUNK, STREAM_RING,
                                                        _host_ptr(host) if host is not None else None, C.byref(k)))
        return host, _fetch_pulses(ctx, k.value)
    d_iq = samples if on_device else to_device(samples, ctx)
    qad = DeviceArray(ctx, (n,), np.float32) if return_qad else None
    ctx.check(
        ctx.lib.urh_demod_digitize(
            ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(d_iq.dtype), n, float(noise_mag), code if code >= 0 else 99,
            float(center), int(tolerance), int(samples_per_symbol), int(bits_per_symbol), float(center_spacing),
            C.c_void_p(qad.ptr if qad is not None else 0), C.byref(k),
        )
    )
    rows = _fetch_pulses(ctx, k.value)
    if qad is not None and not on_device:
        qad = qad.get()
    return qad, rows


def demod_center_digitize(samples, noise_mag: float, mod_type: str, tolerance: int, samples_per_symbol: int,
                          bits_per_symbol: int = 1, center_spacing: float = 0.1, max_size=None, return_qad: bool = False,
                          stepwise: bool = False, out=None, rows_out=None, scratch=None, chunk_samples: int = 1 << 24):
    """afp_demod -> detect_center -> grab_pulse_lens for a capture whose center is not known yet (ASK/FSK): three passes
    over sample-rate data instead of the reference's five (demod + tile statistics, histogram of qad, digitize from qad).
    Binary symbols run as ONE library call (urh_demod_center_digitize): bin edges, histogram, peak pick and the pulse table
    are chained on the device and the host synchronises once.  ``stepwise`` (or a tie the device must not break, or
    bits_per_symbol > 1) takes the call-by-call path with the peak pick in numpy.
    Returns (center, int64[k,2]) or (center, rows, qad) with return_qad.  center None -> no pulses (empty table)."""
    from urh_b200.ainterpretation.AutoInterpretation import demod_detect_center
    on_device = isinstance(samples, DeviceArray)
    code = _lib.demod_mod_code(mod_type)
    one_call = not stepwise and bits_per_symbol == 1 and code in (_lib.MOD_ASK, _lib.MOD_FSK) and len(samples) > 2
    qad = out
    if one_call:
        samples = _check_iq(samples)
        ctx = samples.ctx if on_device else _lib.default_context()
        n = len(samples)
        if qad is None:
            qad = DeviceArray(ctx, (n,), np.float32)
        center, state, k = C.c_double(0.0), C.c_int(0), C.c_int64(0)
        if on_device:
            d_iq = samples
            ctx.check(ctx.lib.urh_demod_center_digitize(ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(d_iq.dtype), n, float(noise_mag),
                                                        code, int(tolerance), int(samples_per_symbol), -1 if max_size is None else int(max_size),
                                                        C.c_void_p(qad.ptr), C.byref(center), C.byref(state), C.byref(k)))
        elif scratch is None and use_stream(n, samples.dtype, tolerance, _lib.STREAM_DEMOD_CENTER_DIGITIZE, device_budget(ctx)):
            return _demod_center_digitize_stream(ctx, samples, noise_mag, code, tolerance, samples_per_symbol, max_size, qad, return_qad,
                                                 rows_out)
        else:
            host = np.ascontiguousarray(samples)
            d_iq = scratch if scratch is not None else DeviceArray(ctx, host.shape, host.dtype)
            ctx.check(ctx.lib.urh_demod_center_digitize_host(ctx.handle, host.ctypes.data_as(C.c_void_p), _lib.dtype_code(host.dtype), n,
                                                             float(noise_mag), code, int(tolerance), int(samples_per_symbol),
                                                             -1 if max_size is None else int(max_size), int(chunk_samples), C.c_void_p(d_iq.ptr),
                                                             C.c_void_p(qad.ptr), C.byref(center), C.byref(state), C.byref(k)))
            samples = d_iq   # the capture is on the device now (the stepwise fallback below reuses it)
        if state.value != 2:
            c = float(center.value) if state.value == 1 else None
            rows = _fetch_pulses(ctx, k.value, rows_out) if c is not None else np.zeros((0, 2), dtype=np.int64)
            if return_qad:
                return c, rows, (qad if on_device else qad.get())
            return c, rows
    qad, center = demod_detect_center(samples, noise_mag, mod_type, max_size, out=qad)
    if center is None:
        rows = np.zeros((0, 2), dtype=np.int64)
    else:
        rows = grab_pulse_lens(qad, float(center), tolerance, mod_type, samples_per_symbol, bits_per_symbol, center_spacing)
    if return_qad:
        return center, rows, (qad if on_device else qad.get())
    return center, rows


def _demod_center_digitize_stream(ctx, samples, noise_mag, code, tolerance, samples_per_symbol, max_size, qad, return_qad, rows_out):
    """demod_center_digitize for a host capture that does not fit: IQ streamed, qad resident (and mirrored to the host with
    return_qad).  A center the device must not decide (state 2) is finished stepwise from the resident qad and the demodulator's
    tile table, as demod_detect_center would, with the digitizer streamed over the resident qad."""
    from urh_b200.ainterpretation import AutoInterpretation as AI
    n = len(samples)
    host = np.empty(n, dtype=np.float32) if return_qad else None
    center, state, kept, k = C.c_double(0.0), C.c_int(0), C.c_int64(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_demod_center_digitize_stream(ctx.handle, _host_ptr(samples), _lib.dtype_code(samples.dtype), n, float(noise_mag),
                                                       code, int(tolerance), int(samples_per_symbol), -1 if max_size is None else int(max_size),
                                                       STREAM_CHUNK, STREAM_RING, C.c_void_p(qad.ptr),
                                                       _host_ptr(host) if host is not None else None, C.byref(center), C.byref(state),
                                                       C.byref(kept), C.byref(k)))
    if state.value == 2:
        st = AI.fused_window_stats(ctx, qad, n, kept.value, max_size)
        c = AI._center_from_stats(ctx, qad, n, st, ctx.lib.urh_center_histogram_tiles)
        rows = np.zeros((0, 2), dtype=np.int64)
        if c is not None:
            ctx.check(ctx.lib.urh_grab_pulse_lens_stream(ctx.handle, C.c_void_p(qad.ptr), 1, n, float(c), int(tolerance), code,
                                                         int(samples_per_symbol), 1, 0.1, STREAM_CHUNK, STREAM_RING, C.byref(k)))
            rows = _fetch_pulses(ctx, k.value, rows_out)
    else:
        c = float(center.value) if state.value == 1 else None
        rows = _fetch_pulses(ctx, k.value, rows_out) if c is not None else np.zeros((0, 2), dtype=np.int64)
    if return_qad:
        return c, rows, host
    return c, rows


def ppseq_to_bits(ppseq, samples_per_symbol: int, bits_per_symbol: int = 1, write_bit_sample_pos: bool = True,
                  pause_threshold: int = 8, ctx=None):
    """ProtocolAnalyzer._ppseq_to_bits (ProtocolAnalyzer.py:323-414) on the GPU.  ``ppseq``: int64[k,2] numpy array or
    DeviceArray, or an int k = "the first k rows of the table the last digitizer call left on the device" (no copy).
    Returns flat arrays: (bits uint8[B], msg_off int64[M+1], pauses int64[M], pos int64[P] or None); message m is
    bits[msg_off[m]:msg_off[m+1]], its bit_sample_pos pos[msg_off[m] + 2m : msg_off[m+1] + 2m + 2] (the last message has
    one trailing entry instead of two when no pause row closes it)."""
    if isinstance(ppseq, (int, np.integer)):
        ctx = ctx or _lib.default_context()
        ptr, k = 0, int(ppseq)
    elif isinstance(ppseq, DeviceArray):
        ctx, ptr, k = ppseq.ctx, ppseq.ptr, len(ppseq)
        if ppseq.dtype != np.int64:
            raise ValueError("pulse table must be int64[k, 2]")
    else:
        rows = np.ascontiguousarray(ppseq, dtype=np.int64).reshape(-1, 2)
        ctx = ctx or _lib.default_context()
        k = len(rows)
        keep = to_device(rows, ctx) if k else None
        ptr = keep.ptr if k else 0
        if k == 0:
            return np.zeros(0, np.uint8), np.zeros(1, np.int64), np.zeros(0, np.int64), (np.zeros(0, np.int64) if write_bit_sample_pos else None)
    m, b, p = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_ppseq_to_bits(ctx.handle, C.c_void_p(ptr), k, int(samples_per_symbol), int(bits_per_symbol), int(pause_threshold),
                                        int(bool(write_bit_sample_pos)), C.byref(m), C.byref(b), C.byref(p)))
    bits = np.empty(b.value, np.uint8)
    off = np.zeros(m.value + 1, np.int64)
    pauses = np.empty(m.value, np.int64)
    pos = np.empty(p.value, np.int64) if write_bit_sample_pos else None
    ctx.check(ctx.lib.urh_fetch_bits(ctx.handle, bits.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p),
                                     pauses.ctypes.data_as(C.c_void_p), pos.ctypes.data_as(C.c_void_p) if pos is not None else None))
    return bits, off, pauses, pos


# ---- modulator ------------------------------------------------------------------------------------------------
def get_oqpsk_bits(original_bits) -> np.ndarray:
    """signal_functions.pyx:179-193 (host; a bit shuffle on a few thousand bits)."""
    bits = np.asarray(original_bits, dtype=np.uint8)
    n = len(bits)
    if n == 0:
        return np.zeros(0, dtype=np.uint8)
    out = np.zeros(n + 2, dtype=np.uint8)
    out[0] = bits[0]
    out[n + 1] = bits[n - 1]
    idx = np.arange(2, n - 2, 2)
    out[idx] = bits[idx]
    out[idx + 1] = bits[idx - 1]
    return out


def gauss_fir(sample_rate: float, samples_per_symbol: int, bt: float = 0.5, filter_width: float = 1.0) -> np.ndarray:
    """signal_functions.pyx:228-243 — Gaussian FIR taps (a few hundred values, host numpy exactly as the reference)."""
    sample_rate = np.float32(sample_rate)
    bt = np.float32(bt)
    filter_width = np.float32(filter_width)
    k = np.arange(-int(filter_width * samples_per_symbol), int(filter_width * samples_per_symbol) + 1, dtype=np.float32)
    ts = np.float32(np.float32(samples_per_symbol) / sample_rate)
    h = (np.sqrt((2 * np.pi) / (np.log(2))) * bt / ts
         * np.exp(-(((np.sqrt(2) * np.pi) / np.sqrt(np.log(2)) * bt * k / samples_per_symbol) ** 2))).astype(np.float32)
    return h / h.sum()


_MOD_CODES = {"ask": _lib.MOD_ASK, "fsk": _lib.MOD_FSK, "psk": _lib.MOD_PSK, "gfsk": _lib.MOD_GFSK, "oqpsk": _lib.MOD_OQPSK}


def modulate_batch(messages, samples_per_symbol, modulation_type, parameters, bits_per_symbol, carrier_amplitude,
                   carrier_frequency, carrier_phase, sample_rate, pauses, start=0, dtype=np.float32, gauss_bt=0.5,
                   filter_width=1.0, device_result=False):
    """Modulate a batch of bit arrays that share one parameter set in ONE launch sequence (addition to the reference API; per message
    the result equals modulate_c(bits, ..., pause, start)).  Returns a list of (total,2) arrays (or one DeviceArray +
    offsets when device_result=True)."""
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype(np.int8), np.dtype(np.int16), np.dtype(np.float32)):
        raise ValueError("Unsupported dtype for modulation {}".format(dtype))
    mod = modulation_type.lower()
    assert mod in _MOD_CODES
    if mod == "oqpsk":
        assert bits_per_symbol == 2
    ctx = _lib.default_context()
    rect = isinstance(messages, np.ndarray) and messages.ndim == 2 and mod != "oqpsk"
    if rect:
        # equal-length messages given as one [nmsg, nbits] array: no per-message Python work
        flat = np.ascontiguousarray(messages, dtype=np.uint8)
        nmsg, per = flat.shape
        pauses = np.asarray(pauses if hasattr(pauses, "__len__") else [pauses] * nmsg, dtype=np.int64)
        bit_off = np.arange(nmsg + 1, dtype=np.int64) * per
        out_off = np.zeros(nmsg + 1, dtype=np.int64)
        np.cumsum(int(per // bits_per_symbol) * int(samples_per_symbol) + pauses, out=out_off[1:])
        msgs = None
    else:
        # ragged batch: per-message Python work only where it is unavoidable (lists -> arrays, the OQPSK bit shuffle);
        # lengths and offsets are vectorised
        msgs = []
        for bits in messages:
            b = bits if (isinstance(bits, np.ndarray) and bits.dtype == np.uint8 and bits.ndim == 1) else \
                np.ascontiguousarray(np.asarray(bits, dtype=np.uint8))
            if mod == "oqpsk" and len(b):
                b = np.ascontiguousarray(get_oqpsk_bits(b)[: len(b)])  # only the first len(bits) shuffled bits are used
            msgs.append(b)
        nmsg = len(msgs)
        pauses = np.asarray(pauses if hasattr(pauses, "__len__") else [pauses] * nmsg, dtype=np.int64)
        lens = np.fromiter((len(b) for b in msgs), dtype=np.int64, count=nmsg)
        bit_off = np.zeros(nmsg + 1, dtype=np.int64)
        np.cumsum(lens, out=bit_off[1:])
        out_off = np.zeros(nmsg + 1, dtype=np.int64)
        np.cumsum((lens // int(bits_per_symbol)) * int(samples_per_symbol) + pauses, out=out_off[1:])
    total = int(out_off[-1])
    params = np.ascontiguousarray(np.asarray(parameters, dtype=np.float32))
    d_out = DeviceArray(ctx, (total, 2), dtype)
    if total and bit_off[-1] > 0:
        d_bits = to_device(flat.reshape(-1) if rect else (np.concatenate(msgs) if nmsg else np.zeros(0, np.uint8)), ctx)
        gfir = gauss_fir(sample_rate, samples_per_symbol, bt=gauss_bt, filter_width=filter_width) if mod == "gfsk" else None
        ctx.check(ctx.lib.urh_modulate_batch(
            ctx.handle, C.c_void_p(d_bits.ptr), bit_off.ctypes.data_as(C.c_void_p), out_off.ctypes.data_as(C.c_void_p), nmsg,
            int(samples_per_symbol), _MOD_CODES[mod], params.ctypes.data_as(C.c_void_p), len(params), int(bits_per_symbol),
            float(carrier_amplitude), float(carrier_frequency), float(carrier_phase), float(sample_rate), int(start),
            _lib.dtype_code(dtype), gfir.ctypes.data_as(C.c_void_p) if gfir is not None else None,
            len(gfir) if gfir is not None else 0, C.c_void_p(d_out.ptr)))
    elif total:
        d_out.zero()
    if device_result:
        return d_out, out_off
    host = d_out.get()
    return [host[out_off[m]: out_off[m + 1]] for m in range(nmsg)]


def modulate_c(bits, samples_per_symbol, modulation_type, parameters, bits_per_symbol, carrier_amplitude,
               carrier_frequency, carrier_phase, sample_rate, pause, start, dtype=np.float32, gauss_bt=0.5, filter_width=1.0):
    """signal_functions.pyx:56-177 — one message."""
    dtype_np = np.dtype(dtype) if dtype in (np.int8, np.int16, np.float32) or isinstance(dtype, np.dtype) else None
    if dtype_np is None or dtype_np not in (np.dtype(np.int8), np.dtype(np.int16), np.dtype(np.float32)):
        raise ValueError("Unsupported dtype for modulation {}".format(dtype))
    bits = np.asarray(bits, dtype=np.uint8)
    if len(bits) == 0:
        return np.zeros((int(pause), 2), dtype=dtype_np)
    assert modulation_type.lower() in _MOD_CODES
    return modulate_batch([bits], samples_per_symbol, modulation_type, parameters, bits_per_symbol, carrier_amplitude,
                          carrier_frequency, carrier_phase, sample_rate, [pause], start, dtype_np, gauss_bt, filter_width)[0]


# ---- filters ----------------------------------------------------------------------------------------------------
def fir_filter(input_samples, filter_taps):
    """signal_functions.pyx:513-525 — causal complex64 FIR, exact accumulation order."""
    on_device = isinstance(input_samples, DeviceArray)
    ctx = input_samples.ctx if on_device else _lib.default_context()
    if not on_device:
        if not isinstance(input_samples, np.ndarray) or input_samples.dtype != np.complex64 or input_samples.ndim != 1:
            raise ValueError("Buffer dtype mismatch, expected 'float complex'")
        input_samples = np.ascontiguousarray(input_samples)
    taps = np.ascontiguousarray(np.asarray(filter_taps, dtype=np.complex64))
    n = len(input_samples)
    if len(taps) == 0:
        # the reference returns np.zeros(N + M - 1)[:N]: N - 1 zeros without taps, and np.zeros(-1) raises for N = 0
        if n == 0:
            raise ValueError("negative dimensions are not allowed")
        if not on_device:
            return np.zeros(n - 1, dtype=np.complex64)
        out = DeviceArray(ctx, (n - 1,), np.complex64)
        return out.zero() if n > 1 else out
    if not on_device and n and filter_use_stream(_lib.FILTER_FIR, n, n, np.float32, len(taps), 0, device_budget(ctx)):
        host = np.empty(n, dtype=np.complex64)
        ctx.check(ctx.lib.urh_fir_filter_stream(ctx.handle, _host_ptr(input_samples), n, _host_ptr(taps) if len(taps) else None, len(taps),
                                                FILTER_STREAM_CHUNK, STREAM_RING, _host_ptr(host)))
        return host
    out = DeviceArray(ctx, (n,), np.complex64)
    if n:
        d = input_samples if on_device else to_device(input_samples.view(np.float32), ctx)
        d_t = to_device(taps.view(np.float32) if len(taps) else np.zeros(2, np.float32), ctx)
        ctx.check(ctx.lib.urh_fir_filter(ctx.handle, C.c_void_p(d.ptr), n, C.c_void_p(d_t.ptr), len(taps), C.c_void_p(out.ptr)))
    return out if on_device else out.get()


def iir_filter(a, b, signal):
    """signal_functions.pyx:527-542 — only caller is an exploratory test script; serial recurrence on tiny inputs."""
    raise NotImplementedError("iir_filter has no caller on the IQ hot path (SURVEY §8b)")


def find_nearest_center(sample: float, centers, num_centers: int) -> int:
    """signal_functions.pyx:497-511 (no caller in the reference)."""
    best, best_d = 0, np.float32(99999)
    for i in range(num_centers):
        d = np.float32((np.float32(sample) - np.float32(centers[i])) ** 2)
        if d < best_d:
            best_d, best = d, i
    return best
