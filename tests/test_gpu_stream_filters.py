"""GPU: host captures streamed through the windowed ring (urh_convolve_c128_stream, urh_fir_filter_stream, urh_dc_correction_stream,
urh_stft_stream, urh_spectrogram_db_stream, urh_spectrogram_bgra_stream; DESIGN.md §4.11) give the resident results word for word, at
small sizes with small chunks; the shims take the streamed path exactly when the resident call does not fit the device budget."""
import ctypes as C

import numpy as np
import pytest


pytestmark = pytest.mark.gpu


def _lib():
    from urh_b200 import _lib as L

    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def capture(n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = np.exp(2j * np.pi * 0.05 * t) * (1 + 0.5 * (rng.random(n) > 0.5)) + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return np.ascontiguousarray(x.astype(np.complex64))


def _stream_stats(ctx):
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_stream_stats(ctx.handle, st))
    return list(st)


# ---- the entries, called with an explicit chunk and ring ------------------------------------------------------------------------------
def s_convolve(ctx, x, taps, offset, out_len, cs, ring=2):
    y = np.full(out_len, np.nan, dtype=np.complex64)   # sentinels: every output is written
    ctx.check(ctx.lib.urh_convolve_c128_stream(ctx.handle, _ptr(x), len(x), _ptr(taps), len(taps), offset, out_len, cs, ring, _ptr(y)))
    return y


def s_fir(ctx, x, taps, cs, ring=2):
    y = np.full(len(x), np.nan, dtype=np.complex64)
    ctx.check(ctx.lib.urh_fir_filter_stream(ctx.handle, _ptr(x), len(x), _ptr(taps) if len(taps) else None, len(taps), cs, ring, _ptr(y)))
    return y


def s_dc(ctx, x, exact, cs, ring=2):
    y = np.full(x.shape, np.nan, dtype=np.float32 if x.dtype == np.float32 else np.float64)
    ctx.check(ctx.lib.urh_dc_correction_stream(ctx.handle, _ptr(x), _lib().dtype_code(x.dtype), len(x), int(exact), cs, ring, _ptr(y)))
    return y


def s_frames(ctx, x, W, hop, frames, mode, cs, ring=2):
    w = np.hanning(W).astype(np.float64)
    out = np.full((frames, W), np.nan, dtype=np.complex128 if mode == 0 else np.float32)
    call = ctx.lib.urh_stft_stream if mode == 0 else ctx.lib.urh_spectrogram_db_stream
    ctx.check(call(ctx.handle, _ptr(x), len(x), W, hop, _ptr(w), frames, cs, ring, _ptr(out)))
    return out


def r_convolve(ctx, x, taps, offset, out_len):
    from urh_b200.device import DeviceArray, to_device

    d_x, d_t = to_device(x.view(np.float32), ctx), to_device(taps.view(np.float64), ctx)
    out = DeviceArray(ctx, (out_len,), np.complex64)
    ctx.check(ctx.lib.urh_convolve_c128(ctx.handle, C.c_void_p(d_x.ptr), len(x), C.c_void_p(d_t.ptr), len(taps), offset, out_len,
                                        C.c_void_p(out.ptr)))
    return out.get()


# ---- band-pass --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bw", sorted(__import__("urh_b200.signalprocessing.Filter", fromlist=["Filter"]).Filter.BANDWIDTHS.values()))
def test_bandpass_presets(ctx, bw):
    from urh_b200.signalprocessing.Filter import Filter

    taps = np.ascontiguousarray(Filter.bandpass_taps(-0.1, 0.2, bw), dtype=np.complex128)
    m = len(taps)   # 11 .. 4001: the tiled kernel (<= 768 taps) and the untiled one
    n = 3 * m + 2 * 1280 + 7
    x = capture(n, m)
    half = (m - 1) // 2
    ref = r_convolve(ctx, x, taps, half, n)
    for cs in (max(1, m // 2), m, 3 * m + 11):
        assert same(s_convolve(ctx, x, taps, half, n, cs), ref), (m, cs)
    for offset, out_len in ((0, n + m - 1), (m - 1, n), (n + m - 5, 2 * m + 9)):   # the last runs past n + m - 1
        assert same(s_convolve(ctx, x, taps, offset, out_len, max(1, m // 3), 3), r_convolve(ctx, x, taps, offset, out_len)), (m, offset)


# ---- FIR --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 10, 101, 1000])
def test_fir(ctx, m):
    from urh_b200.cythonext import signal_functions as sf

    rng = np.random.default_rng(m)
    n = 70_001
    x = capture(n, m + 1)
    taps = np.ascontiguousarray(((rng.standard_normal(m) + 1j * rng.standard_normal(m)) / m).astype(np.complex64))
    ref = sf.fir_filter(x, taps)
    for cs in (1, 999, 4096 + 3, 1 << 20):   # chunks shorter than the history grow to it
        assert same(s_fir(ctx, x, taps, cs, 2 if cs < 4096 else 3), ref), (m, cs)


# ---- DC correction ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1 << 22, (1 << 22) + 1])
def test_dc_float32(ctx, n):
    from urh_b200.signalprocessing.Filter import Filter

    rng = np.random.default_rng(n)
    x = np.ascontiguousarray((rng.standard_normal((n, 2)) * 2 + np.array([0.3, -0.7])).astype(np.float32))
    exact = n <= Filter.EXACT_DC_MAX
    got = s_dc(ctx, x, exact, 1 << 20 if n > 1 else 1)
    if exact:
        assert same(got, Filter.dc_correction(x))
    else:
        assert same(got, x - np.mean(x.astype(np.float64), axis=0).astype(np.float32))


def test_dc_double_regime(ctx):
    n = 5_000_000
    rng = np.random.default_rng(5)   # the data of test_dc_split_double_regime: the mean lies far from a float32 rounding midpoint
    x = np.ascontiguousarray((rng.standard_normal((n, 2)) + np.array([0.123, -0.456])).astype(np.float32))
    ref = x - np.mean(x.astype(np.float64), axis=0).astype(np.float32)
    for cs in (1 << 20, 999_999):
        assert same(s_dc(ctx, x, 0, cs, 3), ref)


@pytest.mark.parametrize("dtype", [np.int8, np.uint8, np.int16, np.uint16])
def test_dc_integer(ctx, dtype):
    from urh_b200.signalprocessing.Filter import Filter

    info = np.iinfo(dtype)
    n = 300_007
    x = np.ascontiguousarray(np.random.default_rng(3).integers(info.min, info.max + 1, (n, 2)).astype(dtype))
    ref = Filter.dc_correction(x)
    for cs in (1, 4096, 100_000):
        assert same(s_dc(ctx, x[: 50] if cs == 1 else x, 0, cs), Filter.dc_correction(x[:50]) if cs == 1 else ref), (dtype, cs)


# ---- STFT / dB map ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [128, 256, 512, 1024, 2048, 4096, 1000, 1001])
@pytest.mark.parametrize("overlap", [0.0, 0.3, 0.5, 0.75])
def test_stft_and_db(ctx, W, overlap):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    spec = Spectrogram(None, window_size=W, overlap_factor=overlap)
    hop = spec.hop_size
    for n in (W - 3, 7 * hop + W + 5):   # n < W: one zero-padded frame
        x = capture(n, W + n)
        frames = spec._num_frames(n)
        ref0, ref1 = spec.stft(x), spec.calculate_spectrogram(x)
        for cs in (hop, 3 * hop + 1):    # one frame per chunk, three
            assert same(s_frames(ctx, x, W, hop, frames, 0, cs), ref0), (W, overlap, n, cs)
            assert same(s_frames(ctx, x, W, hop, frames, 1, cs, 3), ref1), (W, overlap, n, cs)


# ---- images -----------------------------------------------------------------------------------------------------------------------------
def s_images(ctx, spec, x, segments, transpose, cmap, cs, ring=2):
    W, hop = spec.window_size, spec.hop_size
    frames = [spec._num_frames(ln) for _, ln in segments]
    out = np.full(sum(frames) * W * 4, 0xAB, dtype=np.uint8)
    st = np.array([s for s, _ in segments], np.int64)
    ln = np.array([x for _, x in segments], np.int64)
    w = np.hanning(W).astype(np.float64)
    ctx.check(ctx.lib.urh_spectrogram_bgra_stream(ctx.handle, _ptr(x), len(x), W, hop, _ptr(w), _ptr(st), _ptr(ln), len(segments), _ptr(cmap),
                                                  len(cmap), float(spec.data_min), float(spec.data_max), int(transpose), cs, ring, _ptr(out)))
    imgs, off = [], 0
    for f in frames:
        imgs.append(out[off: off + f * W * 4].reshape((f, W, 4) if transpose else (W, f, 4)))
        off += f * W * 4
    return imgs


@pytest.mark.parametrize("W,overlap", [(256, 0.5), (1024, 0.5), (1000, 0.75)])
def test_image_segments(ctx, W, overlap):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    hop = W - int(overlap * W)
    n = 4100 * hop + 11   # at least four segments of Spectrogram.MAX_LINES_PER_VIEW frames
    x = capture(n, W)
    cmap = np.random.default_rng(4).integers(0, 256, (256, 4)).astype(np.uint8)
    spec = Spectrogram(x, window_size=W, overlap_factor=overlap)
    ref = list(spec.create_image_segments(colormap=cmap))
    segments = [(s, e - s) for s, e, _ in spec.segment_bounds()]
    assert len(ref) >= 4
    seg_len = segments[0][1]
    for cs in (seg_len // 3, seg_len + 17, 3 * seg_len):   # pieces of a segment, one segment, several per chunk
        got = s_images(ctx, spec, x, segments, False, cmap, cs)
        assert len(got) == len(ref) and all(same(a, b) for a, b in zip(got, ref)), (W, cs)


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("W", [1024, 1000])
def test_split_single_image(ctx, transpose, W):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n = 200_003
    x = capture(n, 7)
    cmap = np.random.default_rng(5).integers(0, 256, (300, 4)).astype(np.uint8)
    spec = Spectrogram(x, window_size=W, overlap_factor=0.5)
    ref = spec.create_spectrogram_image(1001, n - 5, transpose=transpose, colormap=cmap)
    seg = [(1001, n - 5 - 1001)]
    # the last two: the segment is a little longer than the chunk but its frames fit one chunk, which then uploads only what they
    # read (less than the segment, (len - W) % hop != 0 here)
    for cs in (spec.hop_size, 10 * spec.hop_size + 3, 50_000, seg[0][1] - 116, seg[0][1] - 3):
        (got,) = s_images(ctx, spec, x, seg, transpose, cmap, cs, 3)
        assert same(got, ref), (transpose, W, cs)


# ---- the shims ----------------------------------------------------------------------------------------------------------------------------
STREAMED = ("urh_convolve_c128_stream", "urh_fir_filter_stream", "urh_dc_correction_stream", "urh_stft_stream", "urh_spectrogram_db_stream",
            "urh_spectrogram_bgra_stream")


@pytest.fixture
def low_budget(monkeypatch, ctx):
    """set_low(): a device budget below every resident call's footprint, and small chunks so that every streamed call has several.
    streamed: how often each windowed entry was called (the library's functions wrapped for the test)."""
    from urh_b200.cythonext import signal_functions as sf

    streamed = {}
    for name in STREAMED:
        fn = getattr(ctx.lib, name)

        def wrapped(*args, _fn=fn, _name=name):
            streamed[_name] = streamed.get(_name, 0) + 1
            return _fn(*args)
        monkeypatch.setattr(ctx.lib, name, wrapped)

    def set_low():
        monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(1 << 20))
        monkeypatch.setattr(sf, "FILTER_STREAM_CHUNK", 1 << 14)
    set_low.streamed = streamed
    return set_low


def _streamed(low_budget, call):
    """call(), and whether it called a windowed entry"""
    before = sum(low_budget.streamed.values())
    out = call()
    return out, sum(low_budget.streamed.values()) > before


def test_shims_stream_below_the_budget(ctx, low_budget):
    from urh_b200.signalprocessing.Filter import Filter, FilterType
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n = 300_007
    x = capture(n, 9)
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))
    i16 = np.ascontiguousarray((iq * 3000).astype(np.int16))
    cmap = np.random.default_rng(6).integers(0, 256, (256, 4)).astype(np.uint8)
    fir = Filter([0.1 + 0.2j, 0.3, -0.05j, 0.2, 0.1], FilterType.custom)
    ma = Filter([1 / 10] * 10, FilterType.moving_average)
    dc = Filter([], FilterType.dc_correction)
    spec = Spectrogram(x, window_size=1024, overlap_factor=0.5)
    calls = {
        "bandpass same": lambda: Filter.apply_bandpass_filter(x, -0.1, 0.2, 0.42),
        "bandpass fft": lambda: Filter.apply_bandpass_filter(x, -0.1, 0.2, 0.01),
        "work fir": lambda: fir.work(x),
        "work moving average": lambda: ma.work(iq),
        "work dc float32": lambda: dc.work(iq),
        "work dc int16": lambda: dc.work(i16),
        "stft": lambda: spec.stft(x),
        "spectrogram": lambda: spec.calculate_spectrogram(),
        "image segments": lambda: list(spec.create_image_segments(colormap=cmap)),
        "image": lambda: spec.create_spectrogram_image(500, n - 3, transpose=True, colormap=cmap),
        # a range a little longer than the shim's chunk (2^14 here) whose frames fit one chunk, in both layouts
        "image just over a chunk": lambda: spec.create_spectrogram_image(700, 700 + (1 << 14) + 116, colormap=cmap),
        "image just over a chunk, transposed": lambda: spec.create_spectrogram_image(700, 700 + (1 << 14) + 116, transpose=True,
                                                                                      colormap=cmap),
    }
    ref = {k: _streamed(low_budget, f) for k, f in calls.items()}
    assert not any(s for _, s in ref.values()), [k for k, (_, s) in ref.items() if s]   # resident-size captures keep the resident path
    low_budget()
    for k, f in calls.items():
        got, streamed = _streamed(low_budget, f)
        assert streamed, k
        r = ref[k][0]
        if isinstance(r, list):
            assert len(got) == len(r) and all(same(a, b) for a, b in zip(got, r)), k
        else:
            assert same(got, r), k


def test_filter_range_streams(ctx, low_budget):
    from urh_b200.signalprocessing.Filter import Filter, FilterType
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.Signal import Signal

    n = 200_001
    x = capture(n, 10)
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))

    def run():
        s = Signal("", "filter_range")
        s.iq_array = IQArray(iq.copy())
        s.noise_threshold = 0.1
        s.modulation_type = "FSK"
        s.qad
        s.filter_range(1000, n - 1000, Filter([1 / 10] * 10, FilterType.moving_average))
        s.filter_range(5000, 150_000, Filter([], FilterType.dc_correction))
        return np.asarray(s.iq_array.data).copy(), np.asarray(s.qad).copy()

    ref, streamed = _streamed(low_budget, run)
    assert not streamed
    low_budget()
    got, streamed = _streamed(low_budget, run)
    assert streamed and {"urh_fir_filter_stream", "urh_dc_correction_stream"} <= set(low_budget.streamed)
    assert same(got[0], ref[0]) and same(got[1], ref[1])


def test_device_input_never_streams(ctx, low_budget):
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import DeviceArray, to_device

    x = capture(50_000, 11)
    taps = np.array([0.5, 0.25j, 0.125], np.complex64)
    ref = sf.fir_filter(x, taps)
    low_budget()
    d = to_device(x.view(np.float32).reshape(-1, 2), ctx)
    d = DeviceArray(ctx, (len(x),), np.complex64, d.ptr, base=d)
    got, streamed = _streamed(low_budget, lambda: sf.fir_filter(d, taps))
    assert isinstance(got, DeviceArray) and not streamed
    assert same(got.get(), ref)


# ---- device memory ----------------------------------------------------------------------------------------------------------------------
def _chunks(entry, n, out_len, p0, p1, cs, segments=None):
    """the chunks urh_stream_windows plans for a call"""
    lib = _lib().load_library()
    st = np.array([s for s, _ in segments] if segments else [0], np.int64)
    ln = np.array([x for _, x in segments] if segments else [0], np.int64)
    count = C.c_int64(0)
    assert lib.urh_stream_windows(entry, n, out_len, p0, p1, cs, _ptr(st), _ptr(ln), len(segments) if segments else 0, None, 0,
                                  C.byref(count)) == 0
    return count.value


def _entry_runs(ctx, n, cs):
    """(entry, p0, p1, out_len, dtype, segments, call) for each streamed entry over a capture of n samples in chunks of cs"""
    from urh_b200.signalprocessing.Filter import Filter

    L = _lib()
    x = capture(n, 12)
    iq16 = np.ascontiguousarray((np.stack([x.real, x.imag], axis=1) * 3000).astype(np.int16))
    taps = np.ascontiguousarray(Filter.bandpass_taps(-0.1, 0.2, 0.08), dtype=np.complex128)
    m = len(taps)
    ftaps = np.ones(10, np.complex64) / 10
    W, hop = 1024, 512
    frames = (n - W) // hop + 1
    cmap = np.random.default_rng(7).integers(0, 256, (256, 4)).astype(np.uint8)
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    spec = Spectrogram(None, window_size=W, overlap_factor=0.5)
    segments = [(s, e - s) for s, e, _ in Spectrogram.segment_bounds_of(n, W, hop, 40)]
    img_frames = sum(f for *_, f in Spectrogram.segment_bounds_of(n, W, hop, 40))
    return [
        (L.FILTER_CONVOLVE, m, (m - 1) // 2, n, np.float32, None, lambda: s_convolve(ctx, x, taps, (m - 1) // 2, n, cs, 3)),
        (L.FILTER_FIR, 10, 0, n, np.float32, None, lambda: s_fir(ctx, x, ftaps, cs, 3)),
        (L.FILTER_DC, 0, 0, n, np.int16, None, lambda: s_dc(ctx, iq16, 0, cs, 3)),
        (L.FILTER_STFT, W, hop, frames, np.float32, None, lambda: s_frames(ctx, x, W, hop, frames, 0, cs, 3)),
        (L.FILTER_DB, W, hop, frames, np.float32, None, lambda: s_frames(ctx, x, W, hop, frames, 1, cs, 3)),
        (L.FILTER_IMAGES, W, hop, img_frames, np.float32, segments, lambda: s_images(ctx, spec, x, segments, False, cmap, cs, 3)),
    ]


def test_device_memory_within_footprint(ctx):
    from urh_b200.cythonext import signal_functions as sf

    n, cs = (1 << 22) + 5, 1 << 18
    ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 1))   # the low point is sampled only while measuring
    try:
        for entry, p0, p1, out_len, dtype, segments, call in _entry_runs(ctx, n, cs):
            ctx.sync()
            free, total = C.c_size_t(0), C.c_size_t(0)
            ctx.check(ctx.lib.urh_mem_get_info(ctx.handle, C.byref(free), C.byref(total)))
            call()
            st = _stream_stats(ctx)
            # the chunks of one pass (the DC correction's two passes cut the capture alike)
            assert st[0] > 0 and st[1] == _chunks(entry, n, out_len, p0, p1, cs, segments) > 1, (entry, st)
            used = free.value - st[0]
            cmap_entries = 256 if entry == _lib().FILTER_IMAGES else 0
            assert used <= sf.filter_footprint(entry, n, out_len, dtype, p0, p1, cs, 3, cmap_entries=cmap_entries), (entry, used)
    finally:
        ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 0))


def test_arena_peak_independent_of_n(ctx):
    cs = 1 << 18
    peaks = {}
    for n in ((1 << 22) + 5, (1 << 24) + 5):
        for entry, *_rest, call in _entry_runs(ctx, n, cs):
            call()
            peaks.setdefault(entry, []).append(_stream_stats(ctx)[2])
    for entry, (small, big) in peaks.items():
        assert small == big, (entry, small, big)
