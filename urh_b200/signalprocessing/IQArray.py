"""``IQArray`` — (n,2) C-contiguous sample container (reference: src/urh/signalprocessing/IQArray.py:11-319).

Same constructor, properties, dtype-conversion rules (pinned by the reference's tests/test_iq_array.py) and
file formats.  `magnitudes` runs on the GPU (util.get_magnitudes); `device()` returns / caches the capture in HBM
so that Signal, Filter and the demodulators do not re-upload it.
"""
import ctypes
import os
import tarfile
import tempfile
import wave

import numpy as np

from ..cythonext.util import get_magnitudes
from ..device import DeviceArray

_INT_TYPES = (np.uint8, np.int8, np.uint16, np.int16)


def _sub_loop_error(data):
    """the exception the reference's export_to_sub loop (IQArray.py:281-304) raises for a capture that is not a non-empty (n, 2)
    array: every sample of a 1-D capture is a numpy.uint8 scalar without len(); after no sample at all, lastvalue was never set"""
    for value in np.zeros(min(len(data), 1), np.uint8):
        len(value)
    if False:
        lastvalue = None
    return lastvalue  # noqa: F821


class IQArray(object):
    def __init__(self, data: np.ndarray, dtype=None, n=None, skip_conversion=False, _owned=False):
        if data is None:
            self.__data = np.zeros((n, 2), dtype, order="C")
        elif skip_conversion:
            self.__data = data
        else:
            self.__data = self.convert_array_to_iq(data)
        assert self.__data.dtype not in (np.complex64, np.complex128)
        self._device = None
        # the caller may keep (and later write) the array it passed in unless we made our own copy
        self._aliased = data is not None and not _owned   # _owned: the caller hands the array over and keeps no reference

    # -- numpy-like access -------------------------------------------------------------------------------------
    # The HBM copy (`device()`) must never go stale.  Every accessor that hands out a WRITABLE numpy view of the samples
    # (`data`, `real`, `imag`, `iq[...]`, `convert_to` of the same dtype — the reference lets callers write through them,
    # e.g. ``iq.data[a:b] = 0``) marks the object as aliased: the view may be written at any later time, so from then on
    # `device()` uploads afresh on every call instead of trusting a cached copy.  Readers inside the package use
    # `_peek()`, a read-only view, and keep the cache.
    def _alias(self):
        self._device = None
        self._aliased = True

    def __getitem__(self, item):
        self._alias()
        return self.__data[item]

    def _peek(self, item=None):
        view = self.__data.view() if item is None else self.__data[item]
        if isinstance(view, np.ndarray):
            view.flags.writeable = False
        return view

    def __setitem__(self, key, value):
        self._device = None
        if isinstance(value, (int, float)):
            self.__data[key] = value
            return
        if isinstance(value, IQArray):
            value = value.data
        if value.dtype == np.complex64 or value.dtype == np.complex128:
            self.real[key] = value.real
            self.imag[key] = value.imag
        elif value.ndim == 2:
            self.__data[key] = value
        else:
            self.__data[key] = value.reshape((-1, 2), order="C")

    def __len__(self):
        return len(self.__data)

    def __eq__(self, other):
        return np.array_equal(self._peek(), other._peek() if isinstance(other, IQArray) else other.data)

    @property
    def num_samples(self):
        return self.__data.shape[0]

    @property
    def minimum(self):
        return self.min_max_for_dtype(self.__data.dtype)[0]

    @property
    def maximum(self):
        return self.min_max_for_dtype(self.__data.dtype)[1]

    @property
    def data(self):
        self._alias()
        return self.__data

    @property
    def real(self):
        self._alias()
        return self.__data[:, 0]

    @real.setter
    def real(self, value):
        self._device = None
        self.__data[:, 0] = value

    @property
    def imag(self):
        self._alias()
        return self.__data[:, 1]

    @imag.setter
    def imag(self, value):
        self._device = None
        self.__data[:, 1] = value

    @property
    def dtype(self):
        return self.__data.dtype

    # -- GPU residency ---------------------------------------------------------------------------------------------
    def device(self):
        """the capture as a DeviceArray (uploaded once, invalidated by in-place edits through this object)"""
        from ..device import to_device

        if self._aliased:
            return to_device(np.ascontiguousarray(self.__data))   # a writable view is out there: never cache
        if self._device is None or len(self._device) != len(self.__data):
            self._device = to_device(np.ascontiguousarray(self.__data))
        return self._device

    @property
    def real_device(self):
        """column I of `device()` as a DeviceColumn; unlike `real` it hands out no writable view, so the HBM copy stays cached"""
        from ..device import DeviceColumn

        return DeviceColumn(self.device(), 0)

    @property
    def imag_device(self):
        """column Q of `device()` as a DeviceColumn (see `real_device`)"""
        from ..device import DeviceColumn

        return DeviceColumn(self.device(), 1)

    def own(self):
        """take a private copy of the samples: no outside view can reach them any more, so `device()` may cache again"""
        self.__data = np.array(self.__data, order="C")
        self._device = None
        self._aliased = False
        return self

    @property
    def magnitudes(self):
        return get_magnitudes(np.ascontiguousarray(self.__data))

    @property
    def magnitudes_normalized(self):
        return self.magnitudes / np.sqrt(self.maximum ** 2.0 + self.minimum ** 2.0)

    def as_complex64(self):
        return self.convert_to(np.float32).flatten(order="C").view(np.complex64)

    def to_bytes(self):
        return self.__data.tobytes()

    def subarray(self, start=None, stop=None, step=None):
        return IQArray(np.array(self._peek(slice(start, stop, step)), order="C"), _owned=True)

    def insert_subarray(self, pos, subarray: np.ndarray):
        self._device = None
        if subarray.ndim == 1:
            if subarray.dtype == np.complex64:
                subarray = subarray.view(np.float32)
            elif subarray.dtype == np.complex128:
                subarray = subarray.view(np.float64)
            subarray = subarray.reshape((-1, 2), order="C")
        self.__data = np.insert(self.__data, pos, subarray, axis=0)

    def apply_mask(self, mask: np.ndarray):
        self._device = None
        self.__data = self.__data[mask]

    # -- dtype conversion (IQArray.py:129-203) -------------------------------------------------------------------------
    def convert_to(self, target_dtype) -> np.ndarray:
        """IQArray.py:127-200.  The element-wise conversion runs on the GPU (convert.cu); the same object is returned when
        the dtype already matches."""
        tgt = np.dtype(target_dtype)
        if tgt == self.__data.dtype:
            self._alias()
            return self.__data
        if tgt not in [np.dtype(t) for t in _INT_TYPES + (np.float32,)]:
            raise ValueError("Data type {} not supported".format(target_dtype))
        if self._device is None and len(self.__data) and self.__data.dtype in [np.dtype(t) for t in _INT_TYPES + (np.float32,)]:
            converted = self._convert_streamed(tgt)
            if converted is not None:
                return converted
        return self.convert_to_device(tgt).get()

    def _convert_streamed(self, tgt):
        """the conversion of a host capture whose resident conversion (capture and output on the device) does not fit the device
        budget, streamed through the device into a new host array (urh_convert_iq_stream, the same elements); else None"""
        from .. import _lib
        from ..cythonext import signal_functions as sf

        ctx = _lib.default_context()
        n = len(self.__data)
        if not sf.filter_use_stream(_lib.FILTER_CONVERT, n, n, self.__data.dtype, _lib.dtype_code(tgt), 0, sf.device_budget(ctx)):
            return None
        src = np.ascontiguousarray(self.__data)
        out = np.empty(src.shape, dtype=tgt)
        ctx.check(ctx.lib.urh_convert_iq_stream(ctx.handle, src.ctypes.data_as(ctypes.c_void_p), _lib.dtype_code(src.dtype),
                                                out.ctypes.data_as(ctypes.c_void_p), _lib.dtype_code(tgt), n, sf.FILTER_STREAM_CHUNK,
                                                sf.STREAM_RING))
        return out

    def convert_to_device(self, target_dtype):
        """the converted capture as a DeviceArray (no download)"""
        import ctypes as C

        from .. import _lib
        from ..device import DeviceArray

        tgt = np.dtype(target_dtype)
        src = self.device()
        if tgt == src.dtype:
            return src
        out = DeviceArray(src.ctx, self.__data.shape, tgt)
        src.ctx.check(src.ctx.lib.urh_convert_iq(src.ctx.handle, C.c_void_p(src.ptr), _lib.dtype_code(src.dtype), C.c_void_p(out.ptr),
                                                  _lib.dtype_code(tgt), int(self.__data.size)))
        return out

    # -- files (IQArray.py:115-127, 205-227, 263-275) -------------------------------------------------------------------
    _EXT = {
        (".complex16u", ".cu8"): np.uint8,
        (".complex16s", ".cs8"): np.int8,
        (".complex32u", ".cu16"): np.uint16,
        (".complex32s", ".cs16"): np.int16,
    }

    @classmethod
    def _dtype_for_filename(cls, filename: str):
        for exts, dt in cls._EXT.items():
            if filename.endswith(exts):
                return dt
        return np.float32

    def tofile(self, filename: str):
        self.convert_to(self._dtype_for_filename(filename)).tofile(filename)

    @staticmethod
    def from_file(filename: str):
        dt = IQArray._dtype_for_filename(filename)
        arr = IQArray(data=np.fromfile(filename, dtype=dt), _owned=True)
        if dt == np.uint8:
            return IQArray(arr.convert_to(np.int8), _owned=True)      # unsigned captures are handled as signed
        if dt == np.uint16:
            return IQArray(arr.convert_to(np.int16), _owned=True)
        return arr

    @staticmethod
    def convert_array_to_iq(arr: np.ndarray) -> np.ndarray:
        if arr.ndim == 1:
            if arr.dtype == np.complex64:
                arr = arr.view(np.float32)
            elif arr.dtype == np.complex128:
                arr = arr.view(np.float64)
            if len(arr) % 2:
                arr = arr[:-1]  # drop a trailing half sample
            return arr.reshape((-1, 2), order="C")
        if arr.ndim == 2:
            return arr
        raise ValueError("Too many dimensions")

    @staticmethod
    def min_max_for_dtype(dtype) -> tuple:
        if dtype in (np.float32, np.float64, np.complex64, np.complex128):
            return -1, 1
        return np.iinfo(dtype).min, np.iinfo(dtype).max

    @staticmethod
    def concatenate(*args):
        return IQArray(data=np.concatenate([a._peek() if isinstance(a, IQArray) else a for a in args[0]]), _owned=True)

    def save_compressed(self, filename):
        with tarfile.open(filename, "w:bz2") as tar_write:
            tmp_name = tempfile.mkstemp()[1]
            self.tofile(tmp_name)
            tar_write.add(tmp_name)
        os.remove(tmp_name)

    def export_to_wav(self, filename, num_channels, sample_rate):
        f = wave.open(filename, "w")
        f.setnchannels(num_channels)
        f.setsampwidth(2)
        f.setframerate(sample_rate)
        f.writeframes(self.convert_to(np.int16))
        f.close()

    # bytes of the .sub body copied from the device and written per step of export_to_sub
    SUB_WRITE_BYTES = 64 << 20

    def export_to_sub(self, filename, frequency=433920000, preset="FuriHalSubGhzPresetOok650Async"):
        """The Flipper Zero RAW file of IQArray.py:275-319: run lengths of convert_to(uint8)[:, 0], signed by value > 127, 512 per
        RAW_Data line.  The body is generated on the device (DESIGN §4.12): from the cached capture or one upload of a host capture
        (urh_sub_export, written in SUB_WRITE_BYTES pieces), or, for a host capture whose resident footprint exceeds the device budget
        (the rule of use_stream, $URH_B200_DEVICE_BUDGET included), streamed through the ring and written to the file piece by piece
        (urh_sub_export_stream).  The reference's exceptions for an empty or 1-D capture are raised before the file is created; a
        failure after it was opened removes it."""
        from .. import _lib
        from ..cythonext import signal_functions as sf

        data = self.__data
        if data.ndim == 2 and len(data):
            if data.dtype not in [np.dtype(t) for t in _INT_TYPES + (np.float32,)]:
                raise NotImplementedError("Conversion from {} to {} not supported", data.dtype, np.uint8)
        else:
            _sub_loop_error(data)
        if data.shape[1] != 2:
            # the reference reads column 0 of rows of any width; the device entries read (n, 2) captures
            col = np.ascontiguousarray(data[:, 0])
            return IQArray(np.stack([col, col], axis=1), _owned=True).export_to_sub(filename, frequency, preset)
        n = len(data)
        code = _lib.dtype_code(data.dtype)
        cached = self._device is not None and len(self._device) == n
        ctx = self._device.ctx if cached else _lib.default_context()
        stream = False
        if not cached:
            fp = ctypes.c_int64(0)
            ctx.check(ctx.lib.urh_sub_export_footprint(n, code, 0, sf.FILTER_STREAM_CHUNK, sf.STREAM_RING, ctypes.byref(fp)))
            stream = fp.value > sf.device_budget(ctx)
        body = None
        nbytes = ctypes.c_int64(0)
        if not stream:
            dev = self.device()
            cap = int(ctx.lib.urh_sub_export_bound(n))
            body = DeviceArray(ctx, (cap,), np.uint8)
        try:
            if body is not None:
                ctx.check(ctx.lib.urh_sub_export(ctx.handle, ctypes.c_void_p(dev.ptr), code, n, ctypes.c_void_p(body.ptr), cap,
                                                 ctypes.byref(nbytes)))
            try:
                with open(filename, "w") as subfile:
                    subfile.write("Filetype: Flipper SubGhz RAW File\n")
                    subfile.write("Version: 1\n")
                    subfile.write("Frequency: {}\n".format(frequency))
                    subfile.write("Preset: {}\n".format(preset))
                    subfile.write("Protocol: RAW")
                    subfile.flush()
                    if body is None:
                        src = np.ascontiguousarray(data)
                        ctx.check(ctx.lib.urh_sub_export_stream(ctx.handle, src.ctypes.data_as(ctypes.c_void_p), code, n, subfile.fileno(),
                                                                sf.FILTER_STREAM_CHUNK, sf.STREAM_RING, ctypes.byref(nbytes)))
                    else:
                        piece = np.empty(min(nbytes.value, self.SUB_WRITE_BYTES), np.uint8)
                        for at in range(0, nbytes.value, len(piece) or 1):
                            m = min(len(piece), nbytes.value - at)
                            ctx.check(ctx.lib.urh_memcpy_d2h(ctx.handle, piece.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(body.ptr + at), m))
                            subfile.buffer.write(piece[:m].data)
                    subfile.buffer.write(b"\n")
            except BaseException:
                if os.path.exists(filename):
                    os.remove(filename)
                raise
        finally:
            if body is not None:
                body.free()
