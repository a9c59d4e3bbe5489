"""``Spectrogram`` numerics (reference: src/urh/signalprocessing/Spectrogram.py:94-206).  STFT + dB on the GPU
(spectrogram.cu: one fused kernel for power-of-two windows, cuFFT for the FFT only otherwise), the BGRA colormap look-up, the
spectrogram images (STFT -> dB -> colormap in one launch for every segment of a capture) and the FTA export.
The QImage wrapping of the reference class is GUI and out of scope (INTEGRATION.md §3 shows the three lines)."""
import ctypes as C
import math

import numpy as np

from .. import _lib
from ..cythonext import signal_functions as sf
from ..device import DeviceArray, PinnedArray, to_device
from .IQArray import IQArray

# BGRA colormap (entries x 4 uint8: blue, green, red, alpha) of create_spectrogram_image / create_image_segments when the call
# names none.  The integration sets it from the reference's urh.colormaps.chosen_colormap_numpy_bgra (INTEGRATION.md §3).
chosen_colormap_numpy_bgra = None
# bytes of FTA records generated per band in export_to_fta: band b is written to the file while band b + 1 is produced, from two
# pinned host buffers of this size
FTA_BAND_BYTES = 64 << 20


class Spectrogram(object):
    MAX_LINES_PER_VIEW = 1000
    DEFAULT_FFT_WINDOW_SIZE = 1024

    def __init__(self, samples: np.ndarray, window_size=DEFAULT_FFT_WINDOW_SIZE, overlap_factor=0.5, window_function=np.hanning):
        self.__samples = np.zeros(1, dtype=np.complex64)
        self.samples = samples
        self.window_size = window_size
        self.overlap_factor = overlap_factor
        self.window_function = window_function
        self.data_min, self.data_max = -140, 10

    @property
    def samples(self):
        return self.__samples

    @samples.setter
    def samples(self, value):
        if isinstance(value, DeviceArray):
            if not ((value.dtype == np.complex64 and value.ndim == 1) or (value.dtype == np.float32 and value.ndim == 2 and value.shape[1] == 2)):
                raise ValueError("device samples must be complex64 (n,) or float32 (n, 2)")
        elif isinstance(value, IQArray):
            value = value.as_complex64()
        elif isinstance(value, np.ndarray) and value.dtype != np.complex64:
            value = IQArray(value).as_complex64()
        elif value is None:
            value = np.zeros(1, dtype=np.complex64)
        self.__samples = value

    @property
    def time_bins(self):
        return int(math.ceil(len(self.samples) / self.hop_size))

    @property
    def freq_bins(self):
        return self.window_size

    @property
    def hop_size(self):
        return self.window_size - int(self.overlap_factor * self.window_size)

    def _num_frames(self, n):
        return max(1, (max(n, self.window_size) - self.window_size) // self.hop_size + 1)

    @staticmethod
    def _device_samples(samples, ctx):
        """(device buffer of the complex64 samples, their number); device samples are used in place"""
        if isinstance(samples, DeviceArray):
            return samples, len(samples)
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        return to_device(x.view(np.float32) if len(x) else np.zeros(2, np.float32), ctx), len(x)

    def _window(self, ctx):
        return to_device(np.ascontiguousarray(self.window_function(int(self.window_size)), dtype=np.float64), ctx)

    def _run(self, samples, mode, keep=False):
        ctx = _lib.default_context()
        W, hop = int(self.window_size), int(self.hop_size)
        if not keep and not isinstance(samples, DeviceArray):
            # a host capture whose resident call does not fit the device budget: frames streamed through the windowed ring
            x = np.ascontiguousarray(samples, dtype=np.complex64)
            n = len(x)
            frames = self._num_frames(n)
            entry = _lib.FILTER_STFT if mode == 0 else _lib.FILTER_DB
            if n and sf.filter_use_stream(entry, n, frames, np.float32, W, hop, sf.device_budget(ctx)):
                out = np.empty((frames, W), dtype=np.complex128 if mode == 0 else np.float32)
                call = ctx.lib.urh_stft_stream if mode == 0 else ctx.lib.urh_spectrogram_db_stream
                w = np.ascontiguousarray(self.window_function(W), dtype=np.float64)
                ctx.check(call(ctx.handle, x.ctypes.data_as(C.c_void_p), n, W, hop, w.ctypes.data_as(C.c_void_p), frames,
                               sf.FILTER_STREAM_CHUNK, sf.STREAM_RING, out.ctypes.data_as(C.c_void_p)))
                return out
            samples = x
        d_x, n = self._device_samples(samples, ctx)
        frames = self._num_frames(n)
        d_w = self._window(ctx)
        if mode == 0:
            out = DeviceArray(ctx, (frames, W), np.complex128)
            ctx.check(ctx.lib.urh_stft(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr), frames, C.c_void_p(out.ptr)))
        else:
            out = DeviceArray(ctx, (frames, W), np.float32)
            ctx.check(ctx.lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr), frames, C.c_void_p(out.ptr)))
        return out if keep else out.get()

    def stft(self, samples: np.ndarray):
        """fft(frames * window) / window_size, complex128 [num_frames, window_size] (Spectrogram.py:94-116)"""
        return self._run(samples, 0)

    def calculate_spectrogram(self, samples: np.ndarray = None) -> np.ndarray:
        """fliplr(arr2decibel(fftshift(stft).astype(complex64))), float32 (Spectrogram.py:156-162)"""
        return self._run(self.samples if samples is None else samples, 1)

    @staticmethod
    def apply_bgra_lookup(data: np.ndarray, colormap, data_min=None, data_max=None, normalize=True) -> np.ndarray:
        """Spectrogram.py:192-206 on the GPU: uint8 [cols, rows, 4] image of ``data.T`` through ``colormap`` (entries x 4 bytes BGRA)"""
        if normalize and (data_min is None or data_max is None):
            raise ValueError("Can't normalize without data min and data max")
        ctx = _lib.default_context()
        on_device = isinstance(data, DeviceArray)
        d = data if on_device else to_device(np.ascontiguousarray(data, dtype=np.float32), ctx)
        rows, cols = d.shape
        cmap = np.ascontiguousarray(colormap, dtype=np.uint8)
        if cmap.ndim != 2 or cmap.shape[1] != 4:
            raise ValueError("colormap must be entries x 4 bytes (blue, green, red, alpha)")
        d_map = to_device(cmap, ctx)
        out = DeviceArray(ctx, (cols, rows, 4), np.uint8)
        ctx.check(ctx.lib.urh_bgra_lookup(ctx.handle, C.c_void_p(d.ptr), rows, cols, C.c_void_p(d_map.ptr), len(cmap),
                                          float(data_min) if normalize else 0.0, float(data_max) if normalize else 1.0, int(bool(normalize)),
                                          C.c_void_p(out.ptr)))
        return out if on_device else out.get()

    # ---- images (Spectrogram.py:164-190) ---------------------------------------------------------------------------------------
    @staticmethod
    def _colormap(colormap):
        cmap = chosen_colormap_numpy_bgra if colormap is None else colormap
        if cmap is None:
            raise ValueError("no colormap: pass one or set Spectrogram.chosen_colormap_numpy_bgra (urh.colormaps.chosen_colormap_numpy_bgra)")
        cmap = np.ascontiguousarray(cmap, dtype=np.uint8)
        if cmap.ndim != 2 or cmap.shape[1] != 4 or len(cmap) == 0:
            raise ValueError("colormap must be entries x 4 bytes (blue, green, red, alpha)")
        return cmap

    def segment_bounds(self):
        """[(start, end, frames)] of the slices create_image_segments renders (Spectrogram.py:183-190, the same float arithmetic)"""
        return self.segment_bounds_of(len(self.samples), self.window_size, self.hop_size, self.MAX_LINES_PER_VIEW)

    @staticmethod
    def segment_bounds_of(n, window_size, hop_size, max_lines=MAX_LINES_PER_VIEW):
        """segment_bounds of a capture of n samples, without the samples (a capture sharded over several GPUs)"""
        time_bins = int(math.ceil(n / hop_size))
        n_segments = max(1, time_bins // max_lines)
        step = time_bins / n_segments
        step = max(1, int((step / hop_size) * hop_size ** 2))

        def frames(length):
            return max(1, (max(length, window_size) - window_size) // hop_size + 1)
        return [(i, min(i + step, n), frames(min(i + step, n) - i)) for i in range(0, n, step)]

    def _images(self, d_x, n, segments, transpose, cmap, ctx):
        """one device call for all (start, length) segments: the uint8 buffer with the images back to back, and their shapes"""
        W, hop = int(self.window_size), int(self.hop_size)
        starts = np.array([s for s, _ in segments], dtype=np.int64)
        lens = np.array([ln for _, ln in segments], dtype=np.int64)
        frames = [self._num_frames(int(ln)) for ln in lens]
        shapes = [((f, W, 4) if transpose else (W, f, 4)) for f in frames]
        out = DeviceArray(ctx, (sum(frames) * W * 4,), np.uint8)
        d_map = to_device(cmap, ctx)
        d_w = self._window(ctx)
        ctx.check(ctx.lib.urh_spectrogram_bgra(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr),
                                               starts.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p), len(segments),
                                               C.c_void_p(d_map.ptr), len(cmap), float(self.data_min), float(self.data_max),
                                               int(bool(transpose)), C.c_void_p(out.ptr)))
        return out, shapes

    def _stream_images(self, x, segments, transpose, cmap, ctx):
        """the images of _images from a host capture (numpy arrays) through the windowed ring, when the resident call does not fit the
        device budget (None: it fits)"""
        W, hop = int(self.window_size), int(self.hop_size)
        frames = [self._num_frames(int(ln)) for _, ln in segments]
        if not len(x) or not sf.filter_use_stream(_lib.FILTER_IMAGES, len(x), sum(frames), np.float32, W, hop, sf.device_budget(ctx),
                                                  cmap_entries=len(cmap)):
            return None
        starts = np.array([s for s, _ in segments], dtype=np.int64)
        lens = np.array([ln for _, ln in segments], dtype=np.int64)
        out = np.empty(sum(frames) * W * 4, dtype=np.uint8)
        w = np.ascontiguousarray(self.window_function(W), dtype=np.float64)
        ctx.check(ctx.lib.urh_spectrogram_bgra_stream(ctx.handle, x.ctypes.data_as(C.c_void_p), len(x), W, hop, w.ctypes.data_as(C.c_void_p),
                                                      starts.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p), len(segments),
                                                      cmap.ctypes.data_as(C.c_void_p), len(cmap), float(self.data_min), float(self.data_max),
                                                      int(bool(transpose)), sf.FILTER_STREAM_CHUNK, sf.STREAM_RING,
                                                      out.ctypes.data_as(C.c_void_p)))
        images, off = [], 0
        for f in frames:
            images.append(out[off: off + f * W * 4].reshape((f, W, 4) if transpose else (W, f, 4)))
            off += f * W * 4
        return images

    @staticmethod
    def _split(out, shapes, on_device):
        """the images of one buffer: DeviceArray views, or numpy views of one download"""
        host = None if on_device else out.get()
        off = 0
        for shape in shapes:
            size = shape[0] * shape[1] * 4
            if on_device:
                yield DeviceArray(out.ctx, shape, np.uint8, out.ptr + off, base=out)
            else:
                yield host[off: off + size].reshape(shape)
            off += size

    def create_spectrogram_image(self, sample_start: int = None, sample_end: int = None, step: int = None, transpose=False,
                                 colormap=None):
        """the uint8 BGRA array [W][frames][4] (transpose: [frames][W][4]) that the reference's create_image wraps in a QImage
        (Spectrogram.py:164-181) of samples[sample_start:sample_end:step]; a DeviceArray when the samples are on the device"""
        cmap = self._colormap(colormap)
        ctx = _lib.default_context()
        samples = self.samples
        on_device = isinstance(samples, DeviceArray)
        if on_device:
            n = len(samples)
            start, stop, st = slice(sample_start, sample_end, step).indices(n)
            count = len(range(start, stop, st))
            if st == 1:
                d_x, seg = samples, (start, count)
            else:   # a strided slice, gathered on the device
                d_x = DeviceArray(ctx, (max(count, 1), 2), np.float32)
                ctx.check(ctx.lib.urh_gather_samples(ctx.handle, C.c_void_p(samples.ptr), n, start, st, count, C.c_void_p(d_x.ptr)))
                n, seg = count, (0, count)
        else:
            x = np.ascontiguousarray(samples[sample_start:sample_end:step], dtype=np.complex64)
            streamed = self._stream_images(x, [(0, len(x))], transpose, cmap, ctx)
            if streamed is not None:
                return streamed[0]
            d_x, n = self._device_samples(x, ctx)
            seg = (0, n)
        out, shapes = self._images(d_x, n, [seg], transpose, cmap, ctx)
        return next(self._split(out, shapes, on_device))

    def create_image_segments(self, colormap=None):
        """the images of Spectrogram.py:183-190 (create_spectrogram_image(i, i + step) per segment), all from one device call"""
        cmap = self._colormap(colormap)
        bounds = self.segment_bounds()
        if not bounds:
            return
        ctx = _lib.default_context()
        segments = [(s, e - s) for s, e, _ in bounds]
        if not isinstance(self.samples, DeviceArray):
            streamed = self._stream_images(np.ascontiguousarray(self.samples, dtype=np.complex64), segments, False, cmap, ctx)
            if streamed is not None:
                yield from streamed
                return
        d_x, n = self._device_samples(self.samples, ctx)   # uploaded once
        out, shapes = self._images(d_x, n, segments, False, cmap, ctx)
        yield from self._split(out, shapes, isinstance(self.samples, DeviceArray))

    # ---- FTA export (Spectrogram.py:118-154) ------------------------------------------------------------------------------------
    @staticmethod
    def fta_dtype(include_amplitude):
        return np.dtype([("f", np.float64), ("t", np.uint32), ("a", np.float32)] if include_amplitude else [("f", np.float64), ("t", np.uint32)])

    @staticmethod
    def fta_check_times(frames, time_width, dtype):
        """raise what the reference's loop raises at its first record whose time int(j * time_width) does not fit a uint32
        (numpy's OverflowError; int() of NaN / inf raises ValueError / OverflowError itself), before any file is opened"""
        with np.errstate(invalid="ignore", over="ignore"):
            p = np.arange(frames, dtype=np.float64) * time_width
            bad = ~np.isfinite(p) | (p >= 4294967296.0) | (p <= -1.0)
        if bad.any():
            j = int(np.argmax(bad))
            rec = np.empty(1, dtype=dtype)
            rec[0] = (0.0, int(j * time_width)) + ((0.0,) if len(dtype.names) == 3 else ())

    def export_to_fta(self, sample_rate, filename: str, include_amplitude=False):
        """Frequency (float64), Time (nanoseconds, uint32)[, Amplitude (float32)] records of every (bin, frame) cell, each repeated 3
        (2) times, as the reference writes them (Spectrogram.py:118-154).  The records are generated on the device in bands of
        FTA_BAND_BYTES and written while the next band is produced; the whole array never exists in memory."""
        W = int(self.window_size)
        n = len(self.samples)
        frames = self._num_frames(n)
        freqs = np.ascontiguousarray(np.fft.fftshift(np.fft.fftfreq(W, 1 / sample_rate)), dtype=np.float64)
        time_width = 1e9 * ((n / sample_rate) / frames)
        dtype = self.fta_dtype(include_amplitude)
        self.fta_check_times(frames, time_width, dtype)
        reps = 3 if include_amplitude else 2
        row_bytes = frames * reps * dtype.itemsize
        rows = max(1, min(W, FTA_BAND_BYTES // row_bytes))
        bands = [(r0, min(rows, W - r0)) for r0 in range(0, W, rows)]
        ctx = _lib.default_context()
        d_db = self._run(self.samples, 1, keep=True)
        d_f = to_device(freqs, ctx)
        d_band = DeviceArray(ctx, (rows * row_bytes,), np.uint8)
        hosts = [PinnedArray(rows * row_bytes, np.uint8, ctx) for _ in range(min(2, len(bands)))]

        def produce(b):
            r0, nr = bands[b]
            ctx.check(ctx.lib.urh_fta_records(ctx.handle, C.c_void_p(d_db.ptr), frames, W, r0, nr, C.c_void_p(d_f.ptr), float(time_width),
                                              int(bool(include_amplitude)), C.c_void_p(d_band.ptr), C.c_void_p(hosts[b % 2].ptr)))

        try:
            with open(filename, "wb") as fh:
                produce(0)
                for b in range(len(bands)):
                    ctx.sync()   # band b is in hosts[b % 2]; nothing after it is queued yet
                    if b + 1 < len(bands):
                        produce(b + 1)
                    fh.write(hosts[b % 2].array[: bands[b][1] * row_bytes])
        finally:
            ctx.sync()
            for h in hosts:
                h.free()
