"""``Filter`` (reference: src/urh/signalprocessing/Filter.py).  Same class / static methods; the convolutions and
the DC correction run on the GPU (filter.cu)."""
import ctypes as C
import math
from enum import Enum

import numpy as np

from .. import _lib, settings
from ..cythonext import signal_functions
from ..device import DeviceArray, to_device


class FilterType(Enum):
    moving_average = "moving average"
    dc_correction = "DC correction"
    custom = "custom"


class Filter(object):
    BANDWIDTHS = {"Very Narrow": 0.001, "Narrow": 0.01, "Medium": 0.08, "Wide": 0.1, "Very Wide": 0.42}
    # up to this many rows the DC correction reproduces numpy's serial float32 column sums bit for bit; beyond it an
    # accurate double reduction is used (the reference's own mean is off by percent there, SURVEY H9)
    EXACT_DC_MAX = 1 << 22

    def __init__(self, taps: list, filter_type: FilterType = FilterType.custom):
        self.filter_type = filter_type
        self.taps = taps

    def work(self, input_signal: np.ndarray) -> np.ndarray:
        if self.filter_type == FilterType.dc_correction:
            return self.dc_correction(input_signal)
        return self.apply_fir_filter(input_signal.flatten())

    @staticmethod
    def dc_correction(input_signal: np.ndarray) -> np.ndarray:
        """input_signal - np.mean(input_signal, axis=0) (Filter.py:32-33)"""
        ctx = _lib.default_context()
        if input_signal.dtype != np.float32:
            # integer captures: numpy promotes to float64 and the column means of integers are exact in double
            x = np.ascontiguousarray(input_signal)
            if x.dtype not in (np.int8, np.uint8, np.int16, np.uint16) or x.ndim != 2 or x.shape[1] != 2:
                raise ValueError("dc_correction expects an (n, 2) capture of int8/uint8/int16/uint16/float32")
            if len(x) == 0:
                return x.astype(np.float64)
            streamed = Filter._dc_correction_stream(x, 1, ctx)
            if streamed is not None:
                return streamed
            d = to_device(x, ctx)
            out = DeviceArray(ctx, x.shape, np.float64)
            ctx.check(ctx.lib.urh_dc_correction_int(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(x.dtype), len(x), C.c_void_p(out.ptr)))
            return out.get()
        ctx = _lib.default_context()
        x = np.ascontiguousarray(input_signal)
        n = len(x)
        if n == 0:
            return x.copy()
        streamed = Filter._dc_correction_stream(x, int(n <= Filter.EXACT_DC_MAX), ctx)
        if streamed is not None:
            return streamed
        d = to_device(x, ctx)
        out = DeviceArray(ctx, x.shape, np.float32)
        ctx.check(ctx.lib.urh_dc_correction(ctx.handle, C.c_void_p(d.ptr), n, C.c_void_p(out.ptr), int(n <= Filter.EXACT_DC_MAX)))
        return out.get()

    @staticmethod
    def _dc_correction_stream(x: np.ndarray, exact_order: int, ctx):
        """dc_correction of a host capture through the windowed ring when the resident call does not fit the device budget (None:
        it fits).  Bit for bit the resident result, except float32 above EXACT_DC_MAX, whose double column sums are added chunk by
        chunk: the mean is float32(float64 mean) there as well."""
        n = len(x)
        if not signal_functions.filter_use_stream(_lib.FILTER_DC, n, n, x.dtype, 0, 0, signal_functions.device_budget(ctx)):
            return None
        out = np.empty(x.shape, dtype=np.float32 if x.dtype == np.float32 else np.float64)
        ctx.check(ctx.lib.urh_dc_correction_stream(ctx.handle, x.ctypes.data_as(C.c_void_p), _lib.dtype_code(x.dtype), n, int(exact_order),
                                                   signal_functions.FILTER_STREAM_CHUNK, signal_functions.STREAM_RING,
                                                   out.ctypes.data_as(C.c_void_p)))
        return out

    def apply_fir_filter(self, input_signal: np.ndarray) -> np.ndarray:
        if input_signal.dtype != np.complex64:
            tmp = np.empty(len(input_signal) // 2, dtype=np.complex64)
            tmp.real = input_signal[0::2]
            tmp.imag = input_signal[1::2]
            input_signal = tmp
        return signal_functions.fir_filter(input_signal, np.array(self.taps, dtype=np.complex64))

    @staticmethod
    def read_configured_filter_bw() -> float:
        bw_type = settings.read("bandpass_filter_bw_type", "Medium", str)
        if bw_type in Filter.BANDWIDTHS:
            return Filter.BANDWIDTHS[bw_type]
        if bw_type.lower() == "custom":
            return settings.read("bandpass_filter_custom_bw", 0.1, float)
        return 0.08

    @staticmethod
    def get_bandwidth_from_filter_length(N):
        return 4 / N

    @staticmethod
    def get_filter_length_from_bandwidth(bw):
        N = int(math.ceil((4 / bw)))
        return N + 1 if N % 2 == 0 else N  # odd length

    @staticmethod
    def _convolve_full_slice(data: np.ndarray, h: np.ndarray, offset: int, out_len: int, fft_branch=False) -> np.ndarray:
        """full_convolution(data, h)[offset : offset + out_len] on the GPU (complex128 taps, double accumulation); a host capture whose
        resident call does not fit the device budget streams through the windowed ring.  fft_branch: the reference transforms the whole
        capture (Filter.py:69-82), so one non-finite sample or tap makes every output NaN + NaN j.  Every sample feeds an output of the
        centred crop and the taps are finite past the first check, so a non-finite output is what flags it (DESIGN.md §4.5)."""
        ctx = _lib.default_context()
        x = np.ascontiguousarray(data, dtype=np.complex64)
        taps = np.ascontiguousarray(h, dtype=np.complex128)
        if fft_branch and not np.isfinite(taps).all():
            return np.full(max(out_len, 0), complex(np.nan, np.nan), dtype=np.complex64)
        if (len(x) and len(taps) and out_len > 0
                and signal_functions.filter_use_stream(_lib.FILTER_CONVOLVE, len(x), out_len, np.float32, len(taps), offset,
                                                       signal_functions.device_budget(ctx))):
            out = np.empty(out_len, dtype=np.complex64)
            ctx.check(ctx.lib.urh_convolve_c128_stream(ctx.handle, x.ctypes.data_as(C.c_void_p), len(x), taps.ctypes.data_as(C.c_void_p),
                                                       len(taps), int(offset), int(out_len), signal_functions.FILTER_STREAM_CHUNK,
                                                       signal_functions.STREAM_RING, out.ctypes.data_as(C.c_void_p)))
            if fft_branch:
                words = out.view(np.float32)
                step = 1 << 22
                if not all(np.isfinite(words[i: i + step]).all() for i in range(0, len(words), step)):
                    out.fill(complex(np.nan, np.nan))
            return out
        d_x = to_device(x.view(np.float32), ctx)
        d_t = to_device(taps.view(np.float64), ctx)
        out = DeviceArray(ctx, (out_len,), np.complex64)
        ctx.check(ctx.lib.urh_convolve_c128(ctx.handle, C.c_void_p(d_x.ptr), len(x), C.c_void_p(d_t.ptr), len(taps), int(offset),
                                            int(out_len), C.c_void_p(out.ptr)))
        if fft_branch:
            flag = to_device(np.zeros(1, np.int32), ctx)
            ctx.check(ctx.lib.urh_nonfinite_flag(ctx.handle, C.c_void_p(out.ptr), int(out_len), C.c_void_p(flag.ptr)))
            ctx.check(ctx.lib.urh_nan_fill_if(ctx.handle, C.c_void_p(out.ptr), int(out_len), C.c_void_p(flag.ptr)))
        return out.get()

    @staticmethod
    def fft_convolve_1d(x: np.ndarray, h: np.ndarray):
        """Filter.py:69-82 — centred crop of the full convolution (the reference computes it with a power-of-two FFT in
        complex128; here it is a direct convolution on the GPU with complex128 taps and double accumulation, returned as
        complex64 — what every reference caller casts the result to (IQArray) — i.e. the values agree to 1e-5 of the signal
        scale, DESIGN.md 4.5, not to float64 precision).  Real x and real h take the reference's rfft / irfft branch: the real
        part, as float64 (float32 when both are float32).  One non-finite sample or tap makes every output NaN, as the transform
        does.  len(h) <= 2 gives too_much == 0 and the reference's ``result[0:-0]`` is EMPTY: reproduced."""
        x, h = np.asarray(x), np.asarray(h)
        real = not (np.iscomplexobj(x) or np.iscomplexobj(h))
        dtype = (np.float32 if x.dtype == h.dtype == np.float32 else np.float64) if real else np.complex64
        n = len(x) + len(h) - 1
        too_much = (n - len(x)) // 2
        if too_much == 0:
            return np.zeros(0, dtype=dtype)
        y = Filter._convolve_full_slice(x, h, too_much, n - 2 * too_much, fft_branch=True)
        return y.real.astype(dtype) if real else y

    @staticmethod
    def bandpass_taps(f_low, f_high, filter_bw=0.08):
        """the taps apply_bandpass_filter designs: edges swapped into order and clamped to [-0.5, 0.5]"""
        if f_low > f_high:
            f_low, f_high = f_high, f_low
        f_low = max(-0.5, min(0.5, f_low))
        f_high = max(-0.5, min(0.5, f_high))
        return Filter.design_windowed_sinc_bandpass(f_low, f_high, filter_bw)

    @staticmethod
    def apply_bandpass_filter(data, f_low, f_high, filter_bw=0.08):
        h = Filter.bandpass_taps(f_low, f_high, filter_bw)
        if len(h) < 8 * math.log(math.sqrt(len(data))):
            # np.convolve(data, h, "same"): centred on the longer operand
            big, small = max(len(data), len(h)), min(len(data), len(h))
            return Filter._convolve_full_slice(data, h, (small - 1) // 2, big)
        return Filter.fft_convolve_1d(data, h)

    @staticmethod
    def design_windowed_sinc_lpf(fc, bw):
        N = Filter.get_filter_length_from_bandwidth(bw)
        h = np.sinc(2 * fc * (np.arange(N) - (N - 1) / 2.0)) * np.blackman(N)
        return h / np.sum(h)  # unity gain

    @staticmethod
    def design_windowed_sinc_bandpass(f_low, f_high, bw):
        f_shift = (f_low + f_high) / 2
        f_c = (f_high - f_low) / 2
        N = Filter.get_filter_length_from_bandwidth(bw)
        return Filter.design_windowed_sinc_lpf(f_c, bw=bw) * np.exp(complex(0, 1) * np.pi * 2 * f_shift * np.arange(0, N, dtype=complex))
