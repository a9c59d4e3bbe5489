"""CUDA drop-in for ``urh.cythonext.auto_interpretation`` (reference: src/urh/cythonext/auto_interpretation.pyx)."""
import ctypes as C

import numpy as np

from .. import _lib
from ..device import DeviceArray, to_device


def segment_messages_from_magnitudes(magnitudes, noise_threshold: float) -> list:
    """auto_interpretation.pyx:55-111 — list of (start, end) tuples."""
    on_device = isinstance(magnitudes, DeviceArray)
    if not on_device:
        magnitudes = np.ascontiguousarray(magnitudes)
    if magnitudes.dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
        raise TypeError("No matching signature found")
    n = len(magnitudes)
    if n == 0:
        return []
    ctx = magnitudes.ctx if on_device else _lib.default_context()
    d = magnitudes if on_device else to_device(magnitudes, ctx)
    k = C.c_int64(0)
    ctx.check(ctx.lib.urh_segment_messages(ctx.handle, C.c_void_p(d.ptr), int(d.dtype == np.float64), n, float(noise_threshold),
                                           C.byref(k)))
    seg = np.empty((k.value, 2), dtype=np.int64)
    ctx.check(ctx.lib.urh_fetch_segments(ctx.handle, seg.ctypes.data_as(C.c_void_p), k.value))
    return [(int(a), int(b)) for a, b in seg]


def get_plateau_lengths(rect_data, center, percentage: int = 25) -> np.ndarray:
    """auto_interpretation.pyx:179-208 — uint64 plateau lengths until `percentage` % of the data is covered."""
    on_device = isinstance(rect_data, DeviceArray)
    n = len(rect_data)
    if n == 0 or center is None:
        return np.array([], dtype=np.uint64)
    ctx = rect_data.ctx if on_device else _lib.default_context()
    d = rect_data if on_device else to_device(np.ascontiguousarray(rect_data, dtype=np.float32), ctx)
    cap = 1 << 16
    while True:
        out = np.empty(cap, dtype=np.uint64)
        k = C.c_int64(0)
        ctx.check(ctx.lib.urh_plateau_lengths(ctx.handle, C.c_void_p(d.ptr), n, float(center), int(percentage),
                                              out.ctypes.data_as(C.c_void_p), cap, C.byref(k)))
        if k.value <= cap:
            return out[: k.value].copy()
        cap = k.value


def merge_plateaus(plateaus, tolerance: int, max_count: int) -> np.ndarray:
    """auto_interpretation.pyx:145-176 — merge plateaus <= tolerance into their neighbours.  The table has at most
    a few thousand entries per message (it is cut at max_count); host arithmetic, like the other per-message glue."""
    plateaus = np.asarray(plateaus, dtype=np.uint64)
    L = len(plateaus)
    if L == 0:
        return np.zeros(0, dtype=np.uint64)
    out = [0 if plateaus[0] <= tolerance else int(plateaus[0])]
    i = 1
    while i < L and len(out) - 1 < max_count:
        if plateaus[i] <= tolerance:
            n = 2
            while i + n < L and plateaus[i + n] <= tolerance:
                n += 2
            out[-1] = int(plateaus[i - 1: min(L, i + n)].sum())
            i += n
        else:
            out.append(int(plateaus[i]))
            i += 1
    return np.array(out, dtype=np.uint64)


def get_threshold_divisor_histogram(plateau_lengths, threshold: float = 0.2) -> np.ndarray:
    """auto_interpretation.pyx:113-143 — for every pair (i < j) of non-zero lengths, count the smaller value if max/min is within
    `threshold` above an integer.  The test depends on the two VALUES only, so the O(L^2) pair loop folds into the (few) distinct
    values with their multiplicities: c_a * c_b pairs for two different values, c_a (c_a - 1) / 2 for a value with itself (whose
    quotient is exactly 1, always counted).  Same counts as the reference's loop; a message with thousands of rounded plateaus
    costs microseconds instead of the quadratic loop (0.2 s per message in the sharded estimate of configs[4])."""
    pl = np.asarray(plateau_lengths, dtype=np.uint64)
    hist = np.zeros(int(np.max(pl)) + 1, dtype=np.uint64)
    if len(pl) < 2:
        return hist
    thr = float(np.float32(threshold))   # the reference compares a double with its float parameter
    u, c = np.unique(pl[pl != 0], return_counts=True)   # ascending
    if len(u) == 0:
        return hist
    c = c.astype(np.uint64)
    hist[u.astype(np.int64)] += c * (c - np.uint64(1)) // np.uint64(2)
    block = 2048   # rows of the value-pair matrix per step (bounded memory for unrounded tables)
    for lo in range(0, len(u) - 1, block):
        mn = u[lo:lo + block, None]
        mx = u[None, :]
        upper = np.arange(len(u))[None, :] > np.arange(lo, min(lo + block, len(u)))[:, None]
        ok = upper & ((mx.astype(np.float64) / mn.astype(np.float64) - (mx // mn).astype(np.float64)) < thr)
        add = (ok * c[None, :]).sum(axis=1, dtype=np.uint64) * c[lo:lo + block]
        hist[u[lo:lo + block].astype(np.int64)] += add
    return hist


def median_filter(data, k: int = 3):
    """auto_interpretation.pyx:211-240 — window [i, i+k) truncated at the end, float32 result."""
    on_device = isinstance(data, DeviceArray)
    ctx = data.ctx if on_device else _lib.default_context()
    if not on_device:
        data = np.ascontiguousarray(data, dtype=np.float64)
    n = len(data)
    out = DeviceArray(ctx, (n,), np.float32)
    if n:
        d = data if on_device else to_device(data, ctx)
        ctx.check(ctx.lib.urh_median_filter(ctx.handle, C.c_void_p(d.ptr), n, int(k), C.c_void_p(out.ptr)))
    return out if on_device else out.get()
