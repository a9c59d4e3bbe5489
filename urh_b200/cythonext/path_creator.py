"""CUDA drop-in for ``urh.cythonext.path_creator`` (reference: src/urh/cythonext/path_creator.pyx).

``create_path_streams`` does the sample-rate work of ``create_path`` on the device: the per-pixel min/max of the visible range
and the QPainterPath byte streams of every sub-path, returned as ``bytes`` (``b""`` for an empty sub-path).  ``create_path``
turns them into ``QPainterPath`` objects exactly as the reference does (``QDataStream(QByteArray) >> path``); PyQt6 is imported
inside that call only, so this module imports without Qt.  Install with
``sys.modules["urh.cythonext.path_creator"] = urh_b200.cythonext.path_creator``.

``samples`` is a 1-D numpy array of int8, uint8, int16, uint16 or float32 (any stride; only ``[start:end]`` is uploaded), a 1-D
``DeviceArray`` or a ``DeviceColumn`` (one column of an (n, 2) capture in HBM, e.g. ``Signal.real_plot_data_device``).
"""
import ctypes as C
import math

import numpy as np

from .. import _lib, settings
from ..device import DeviceArray, DeviceColumn, to_device

# the record of array_to_QPath (path_creator.pyx:102-116): connect flag, x, y, big-endian, packed
_RECORD = np.dtype([("c", ">i4"), ("x", ">f8"), ("y", ">f8")])


def _source(samples, start: int, end: int):
    """(ctx, device source, element stride, n, start, end, keep-alive) with 0 <= start <= end <= n checked"""
    if isinstance(samples, (DeviceArray, DeviceColumn)):
        if samples.ndim != 1:
            raise ValueError("Buffer has wrong number of dimensions (expected 1, got %d)" % samples.ndim)
        if samples.dtype not in _lib._DTYPE_CODE:
            raise TypeError("No matching signature found")
        n = len(samples)
        if not 0 <= start <= end <= n:
            raise ValueError("need 0 <= start <= end <= len(samples), got start=%d end=%d len=%d" % (start, end, n))
        return samples.ctx, samples.ptr, getattr(samples, "stride", 1), n, start, end, samples
    samples = np.asarray(samples)
    if samples.dtype not in _lib._DTYPE_CODE:
        raise TypeError("No matching signature found")
    if samples.ndim != 1:
        raise ValueError("Buffer has wrong number of dimensions (expected 1, got %d)" % samples.ndim)
    n = len(samples)
    if not 0 <= start <= end <= n:
        raise ValueError("need 0 <= start <= end <= len(samples), got start=%d end=%d len=%d" % (start, end, n))
    ctx = _lib.default_context()
    d = to_device(np.ascontiguousarray(samples[start:end]), ctx)   # the visible range only
    return ctx, d.ptr, 1, end - start, 0, end - start, d


def _slice_bounds(subpath_ranges, start, end, scale, length):
    """[lo, hi) of each sub-path into x / values (path_creator.pyx:74-80: Python float arithmetic on the float32 scale), clamped
    as a Python slice of `length` elements"""
    out = np.empty((len(subpath_ranges), 2), dtype=np.int64)
    for k, rng in enumerate(subpath_ranges):
        lo = ((((rng[0] - start) / scale) * scale) - 2 * scale) / scale
        hi = ((((rng[1] - start) / scale) * scale) + 2 * scale) / scale
        out[k, 0] = min(int(max(0, math.floor(lo))), length)
        out[k, 1] = min(int(max(0, math.ceil(hi))), length)
    return out


def create_path_streams(samples, start, end, subpath_ranges=None) -> list:
    """path_creator.pyx:19-82 up to the bytes each sub-path's QPainterPath is read from (array_to_QPath :88-120)"""
    start, end = int(start), int(end)
    ctx, ptr, stride, n, s0, s1, keep = _source(samples, start, end)
    dt = _lib.dtype_code(keep.dtype)
    subpath_ranges = [(start, end)] if subpath_ranges is None else subpath_ranges
    N = end - start
    spp = int(N / settings.PIXELS_PER_PATH)
    values = None
    if spp > 1:
        P = -(-N // spp)
        length = 2 * P
        scale = float(np.float32(N / (2.0 * P)))
        values = DeviceArray(ctx, (length,), keep.dtype)
        ctx.check(ctx.lib.urh_path_minmax(ctx.handle, C.c_void_p(ptr), dt, stride, n, s0, s1, spp, C.c_void_p(values.ptr)))
    else:
        length, scale = N, 1.0
    bounds = _slice_bounds(subpath_ranges, start, end, scale, length)
    count = len(bounds)
    offsets = np.zeros(count + 1, dtype=np.int64)
    vptr = C.c_void_p(values.ptr if values is not None else None)
    args = (ctx.handle, C.c_void_p(ptr), dt, stride, n, s0, s1, spp, start, vptr, bounds.ctypes.data_as(C.c_void_p), count)
    ctx.check(ctx.lib.urh_qpath_streams(*args, None, offsets.ctypes.data_as(C.c_void_p)))
    total = int(offsets[-1])
    if total == 0:
        return [b""] * count
    out = DeviceArray(ctx, (total,), np.uint8)
    ctx.check(ctx.lib.urh_qpath_streams(*args, C.c_void_p(out.ptr), offsets.ctypes.data_as(C.c_void_p)))
    host = out.get().tobytes()   # synchronises
    return [host[offsets[k]:offsets[k + 1]] for k in range(count)]


def _painter_path(stream: bytes):
    from PyQt6.QtCore import QByteArray, QDataStream
    from PyQt6.QtGui import QPainterPath

    path = QPainterPath()
    if stream:
        ds = QDataStream(QByteArray(stream))
        ds >> path
    return path


def create_path(samples, start, end, subpath_ranges=None) -> list:
    """path_creator.pyx:19-82: one QPainterPath per sub-path (needs PyQt6)"""
    import PyQt6.QtCore  # noqa: F401  (ImportError before any device work when Qt is missing)
    import PyQt6.QtGui  # noqa: F401

    return [_painter_path(s) for s in create_path_streams(samples, start, end, subpath_ranges)]


def qpath_stream(x, y) -> bytes:
    """the QDataStream bytes array_to_QPath (path_creator.pyx:88-120) reads a path from, encoded on the host: big-endian
    {i4 n, n x {i4 1, f8 x, f8 -y}, i4 0, i4 0}, y negated in its own dtype; b"" for no points"""
    x = np.asarray(x)
    n = len(x)
    if n == 0:
        return b""
    rec = np.empty(n, dtype=_RECORD)
    rec["c"] = 1
    rec["x"] = x
    with np.errstate(invalid="ignore"):   # a signalling NaN is quieted, as it is in the reference
        rec["y"] = np.negative(np.asarray(y))
    return np.array(n, ">i4").tobytes() + rec.tobytes() + bytes(8)


def array_to_QPath(x, y):
    """path_creator.pyx:88-120 for small host arrays (SceneManager.create_rectangle, Modulator.py:210)"""
    return _painter_path(qpath_stream(x, y))
