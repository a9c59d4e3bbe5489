"""Device-resident arrays (HBM) and pinned host arrays for the GPU hot path."""
import ctypes as C

import numpy as np

from . import _lib


class DeviceArray:
    """A typed, shaped view of device memory owned (or borrowed) by a Context.

    Mirrors the small part of the numpy interface the DSP objects need (shape, dtype, len, slicing
    along axis 0, ``.get()`` to materialise on the host)."""

    def __init__(self, ctx: _lib.Context, shape, dtype, ptr: int = None, base=None):
        self.ctx = ctx
        self.shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize
        self._base = base
        if ptr is None:
            p = C.c_void_p()
            ctx.check(ctx.lib.urh_malloc(ctx.handle, self.nbytes, C.byref(p)))
            self.ptr = p.value
            self._owns = True
        else:
            self.ptr = int(ptr)
            self._owns = False

    def __len__(self):
        return self.shape[0] if self.shape else 0

    @property
    def ndim(self):
        return len(self.shape)

    @property
    def size(self):
        return int(np.prod(self.shape, dtype=np.int64))

    def free(self):
        if self._owns and self.ptr:
            self.ctx.check(self.ctx.lib.urh_free(self.ctx.handle, C.c_void_p(self.ptr)))
            self.ptr = 0
            self._owns = False

    def __del__(self):
        try:
            if self._owns and self.ptr and self.ctx.handle:
                self.ctx.lib.urh_free(self.ctx.handle, C.c_void_p(self.ptr))
        except Exception:
            pass

    def __getitem__(self, item):
        """Contiguous slices along axis 0 only (views, no copy)."""
        if not isinstance(item, slice):
            raise TypeError("DeviceArray supports only axis-0 slices")
        start, stop, step = item.indices(self.shape[0])
        if step != 1:
            raise ValueError("DeviceArray slices must be contiguous")
        stop = max(stop, start)
        row = self.dtype.itemsize * int(np.prod(self.shape[1:], dtype=np.int64))
        return DeviceArray(self.ctx, (stop - start,) + self.shape[1:], self.dtype, self.ptr + start * row, base=self)

    def get(self, out: np.ndarray = None) -> np.ndarray:
        if out is None:
            out = np.empty(self.shape, dtype=self.dtype)
        assert out.nbytes == self.nbytes and out.flags.c_contiguous
        self.ctx.check(self.ctx.lib.urh_memcpy_d2h(self.ctx.handle, out.ctypes.data_as(C.c_void_p), C.c_void_p(self.ptr), self.nbytes))
        return out

    def set(self, host: np.ndarray):
        host = np.ascontiguousarray(host, dtype=self.dtype)
        assert host.nbytes == self.nbytes
        self.ctx.check(self.ctx.lib.urh_memcpy_h2d(self.ctx.handle, C.c_void_p(self.ptr), host.ctypes.data_as(C.c_void_p), self.nbytes))
        self.ctx.sync()  # the host buffer may be pageable / temporary
        return self

    def set_async(self, host: np.ndarray):
        """H2D on the context stream without synchronising (the host array must be pinned and stay alive)."""
        assert host.nbytes == self.nbytes and host.flags.c_contiguous and host.dtype == self.dtype
        self.ctx.check(self.ctx.lib.urh_memcpy_h2d(self.ctx.handle, C.c_void_p(self.ptr), host.ctypes.data_as(C.c_void_p), self.nbytes))
        return self

    def zero(self):
        self.ctx.check(self.ctx.lib.urh_memset(self.ctx.handle, C.c_void_p(self.ptr), 0, self.nbytes))
        return self


class DeviceColumn:
    """A read-only 1-D view of column 0 (I) or 1 (Q) of an ``(n, 2)`` DeviceArray, without a copy.

    What URH's scene code touches of its plot data (``len``, ``dtype``) and what ``path_creator.create_path`` reads on the
    device: element i is ``ptr + i * stride * itemsize``."""

    stride = 2
    ndim = 1

    def __init__(self, array: DeviceArray, column: int):
        if array.ndim != 2 or array.shape[1] != 2 or column not in (0, 1):
            raise ValueError("DeviceColumn needs an (n, 2) DeviceArray and column 0 or 1")
        self.array = array
        self.column = column
        self.ctx = array.ctx
        self.dtype = array.dtype
        self.shape = (array.shape[0],)
        self.ptr = array.ptr + column * array.dtype.itemsize

    def __len__(self):
        return self.shape[0]

    def get(self) -> np.ndarray:
        return np.ascontiguousarray(self.array.get()[:, self.column])


def to_device(arr, ctx: _lib.Context = None) -> DeviceArray:
    if isinstance(arr, DeviceArray):
        return arr
    ctx = ctx or _lib.default_context()
    arr = np.ascontiguousarray(arr)
    d = DeviceArray(ctx, arr.shape, arr.dtype)
    if arr.nbytes:
        d.set(arr)
    return d


def empty(shape, dtype, ctx: _lib.Context = None) -> DeviceArray:
    return DeviceArray(ctx or _lib.default_context(), shape, dtype)


class PinnedArray:
    """Page-locked host memory exposed as a numpy array (``.array``)."""

    def __init__(self, shape, dtype, ctx: _lib.Context = None):
        self.ctx = ctx or _lib.default_context()
        self.dtype = np.dtype(dtype)
        shape = tuple(shape) if isinstance(shape, (tuple, list)) else (int(shape),)
        nbytes = int(np.prod(shape, dtype=np.int64)) * self.dtype.itemsize
        p = C.c_void_p()
        self.ctx.check(self.ctx.lib.urh_host_alloc(self.ctx.handle, max(nbytes, 16), C.byref(p)))
        self.ptr = p.value
        buf = (C.c_char * max(nbytes, 16)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(shape, dtype=np.int64))).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            self.ctx.check(self.ctx.lib.urh_host_free(self.ctx.handle, C.c_void_p(self.ptr)))
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
