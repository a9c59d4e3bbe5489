"""GPU: the kernels that restate the reference's numpy expressions for the capture and image objects, bit for bit against those
expressions evaluated on the host with the reference's argument types (Python-scalar bounds, np.take(mode="clip")):

- the colormap look-up k_bgra_lookup (Spectrogram.apply_bgra_lookup) at every kind of (min, max) bound, non-finite, subnormal and
  huge data, normalize=False indices on both sides of the int64 cast's limits, colormaps on both sides of the shared-memory switch
  and of the fused image kernel's limit, and shapes from 1 x 1 to a grid-stride wrap;
- its copies in the image kernels (k_stft_r16 mode 2, k_bgra_place): create_spectrogram_image and create_image_segments against
  the reference expression applied to the device's own dB map, and the streamed image entry against the resident one;
- the capture conversions k_convert (IQArray.convert_to): every integer source value, float32 values at every truncation and wrap
  boundary, non-finite and huge values, odd counts and offsets, a grid-stride wrap, and the streamed entry;
- the strided sample gather of create_spectrogram_image on device samples, against numpy slicing."""
import ctypes as C

import numpy as np
import pytest

from bgra_restatement import (ALL_RANGES, DECIMAL_RANGES, EQUAL_RANGES, REVERSED_RANGES, SPECIAL_VALUES, TINY_RANGES, boundary_values,
                              device_indices, distinct_colormap, index_values, reference_indices, reference_take)

pytestmark = pytest.mark.gpu

ENTRIES = [1, 2, 256, 1024, 1025, 65536, 65537]
CMAPS = {L: distinct_colormap(L, seed=L) for L in ENTRIES}
INT_TYPES = [np.int8, np.uint8, np.int16, np.uint16]
ALL_TYPES = INT_TYPES + [np.float32]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _first_mismatch(got, want):
    bad = np.argwhere(np.any(got != want, axis=-1))
    return len(bad), bad[:4].tolist()


@pytest.fixture(scope="module")
def sm_count(ctx):
    return ctx.device_info()["sm_count"]


# ---- the colormap look-up (k_bgra_lookup) -------------------------------------------------------------------------------------------
def _lookup(data, cmap, lo=None, hi=None, normalize=True):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    return Spectrogram.apply_bgra_lookup(data, cmap, lo, hi, normalize=normalize)


def _check_lookup(data, L, lo=None, hi=None, normalize=True):
    got = _lookup(data, CMAPS[L], lo, hi, normalize)
    want = reference_take(data, CMAPS[L], lo, hi, normalize)
    assert got.shape == want.shape == (data.shape[1], data.shape[0], 4)
    assert np.array_equal(got, want), (L, lo, hi, normalize, data.shape) + _first_mismatch(got, want)


def _shapes(v):
    """v as one row, one column and a non-square matrix (padded with its own values): a transposition shows in all three"""
    cols = 7 if len(v) > 7 else 2
    m = np.resize(v, (-(-len(v) // cols), cols))
    return [v.reshape(1, -1), v.reshape(-1, 1), m]


@pytest.mark.parametrize("L", ENTRIES)
def test_lookup_every_range_kind(L):
    """integer, float32-exact, decimal (range rounded differently from float32 bounds), 1e-3 wide, min == max and min > max bounds,
    on the data of every index boundary of the range (+-2 ulp) and NaN, +-inf, +-0, subnormals, +-1e30, +-FLT_MAX"""
    for lo, hi in ALL_RANGES:
        v = np.concatenate([boundary_values(lo, hi, L), SPECIAL_VALUES])
        for data in _shapes(v):
            _check_lookup(data, L, lo, hi)
        for x in SPECIAL_VALUES[:6]:   # 1 x 1
            _check_lookup(np.array([[x]], np.float32), L, lo, hi)


@pytest.mark.parametrize("L", ENTRIES)
def test_lookup_indices_without_normalising(L):
    """normalize=False: negative, fractional and >= L indices, 9.0e18 and the float32 below it, 9.1e18, the largest float32 below
    2^63 (all cast exactly by numpy), 2^63 and -2^63, and non-finite values"""
    v = index_values(L)
    for data in _shapes(v):
        _check_lookup(data, L, normalize=False)
    got = _lookup(np.array([[9.1e18, 2.0 ** 63, -(2.0 ** 63)]], np.float32), CMAPS[L], normalize=False)
    assert np.array_equal(got[:, 0], CMAPS[L][[L - 1, 0, 0]])   # numpy: int64(9.1e18) clips to the last entry


@pytest.mark.parametrize("L", [256, 1025])
def test_lookup_grid_stride_wrap(sm_count, L):
    """rows * cols above 2 x (sm_count x 16 blocks of 256 threads): every thread takes three or more pixels"""
    lo, hi = DECIMAL_RANGES[0]
    total = 2 * sm_count * 16 * 256 + 12345
    rows = 1031
    cols = -(-total // rows)
    rng = np.random.default_rng(L)
    data = (rng.uniform(lo - 5, hi + 5, rows * cols)).astype(np.float32)
    b = boundary_values(lo, hi, L)
    data[: len(b)] = b
    data[len(b): len(b) + len(SPECIAL_VALUES)] = SPECIAL_VALUES
    _check_lookup(rng.permutation(data).reshape(rows, cols), L, lo, hi)


# ---- the images: the fused kernel (power-of-two W, up to 65536 entries) and the composed path ---------------------------------------
IMAGE_RANGES = DECIMAL_RANGES[:2] + REVERSED_RANGES + TINY_RANGES + EQUAL_RANGES
IMAGE_ENTRIES = [256, 65536, 65537]


def _capture(n, W, seed=1):
    """a tone with DC, noise from a quarter in, the second half decaying over a few hundred dB, and 2 W exact zeros (-inf frames):
    dB values across every image range"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = (0.25 - 0.5j) + 2.0 * np.exp(2j * np.pi * 0.1937 * t)
    x[n // 4:] += 0.05 * (rng.standard_normal(n - n // 4) + 1j * rng.standard_normal(n - n // 4))
    x[n // 2:] *= np.exp(-np.arange(n - n // 2) / (n / 12))
    x[n // 2 + W // 2: n // 2 + W // 2 + 2 * W] = 0
    return x.astype(np.complex64)


@pytest.mark.parametrize("W", [128, 1024, 1000])
def test_image_against_reference_expression(W):
    """create_spectrogram_image (both layouts) == the reference's expression applied to the device's own calculate_spectrogram()
    map, at decimal, reversed, 1e-3 wide and empty ranges; 65536 entries take the fused kernel at W = 128 / 1024 and 65537 the
    composed path, W = 1000 is composed throughout.  The decimal ranges must pick another entry than the old twice-rounded range
    somewhere on these maps, so that the test sees that arithmetic"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    hop = W // 2
    x = _capture(W + 300 * hop + 17, W, seed=W)
    spec = Spectrogram(x, W, 0.5)
    db = spec.calculate_spectrogram(x)
    separated = 0
    for transpose in (False, True):
        data = np.ascontiguousarray(np.flipud(db.T)) if transpose else db
        for L in IMAGE_ENTRIES:
            for lo, hi in IMAGE_RANGES:
                spec.data_min, spec.data_max = lo, hi
                got = spec.create_spectrogram_image(transpose=transpose, colormap=CMAPS[L])
                want = reference_take(data, CMAPS[L], lo, hi)
                assert got.shape == want.shape and got.dtype == np.uint8, (got.shape, want.shape)
                assert np.array_equal(got, want), (W, transpose, L, lo, hi) + _first_mismatch(got, want)
                if L >= 65536 and (lo, hi) in DECIMAL_RANGES:
                    separated += int(np.any(device_indices(data, L, lo, hi, before_fix=True) != reference_indices(data, L, lo, hi)))
    assert separated == 8, separated


def _segment_capture(W):
    """long enough for two create_image_segments segments at hop W / 2"""
    return _capture(2100 * (W // 2) + W + 5, W, seed=W + 1)


@pytest.mark.parametrize("W", [128, 1024, 1000])
def test_image_segments_against_reference_expression(W):
    """create_image_segments: each segment's image == the reference expression on the device's dB map of that segment"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    x = _segment_capture(W)
    spec = Spectrogram(x, W, 0.5)
    bounds = spec.segment_bounds()
    assert len(bounds) == 2
    dbs = [spec.calculate_spectrogram(x[s:e]) for s, e, _ in bounds]
    for L in (65536, 65537):
        for lo, hi in DECIMAL_RANGES[:2] + REVERSED_RANGES[:1]:
            spec.data_min, spec.data_max = lo, hi
            imgs = list(spec.create_image_segments(colormap=CMAPS[L]))
            assert len(imgs) == len(bounds)
            for (s, e, frames), img, db in zip(bounds, imgs, dbs):
                want = reference_take(db, CMAPS[L], lo, hi)
                assert img.shape == want.shape == (W, frames, 4)
                assert np.array_equal(img, want), (W, L, lo, hi, s) + _first_mismatch(img, want)


def _stream_images(ctx, spec, x, segments, transpose, cmap, chunk):
    W, hop = spec.window_size, spec.hop_size
    frames = [spec._num_frames(ln) for _, ln in segments]
    out = np.full(sum(frames) * W * 4, 0xAB, dtype=np.uint8)
    st = np.array([s for s, _ in segments], np.int64)
    ln = np.array([n for _, n in segments], np.int64)
    w = np.hanning(W).astype(np.float64)
    ctx.check(ctx.lib.urh_spectrogram_bgra_stream(ctx.handle, _ptr(x), len(x), W, hop, _ptr(w), _ptr(st), _ptr(ln), len(segments),
                                                  _ptr(cmap), len(cmap), spec.data_min, spec.data_max, int(transpose), chunk, 2,
                                                  _ptr(out)))
    imgs, off = [], 0
    for f in frames:
        imgs.append(out[off: off + f * W * 4].reshape((f, W, 4) if transpose else (W, f, 4)))
        off += f * W * 4
    return imgs


@pytest.mark.parametrize("W", [1024, 1000])
def test_streamed_images_equal_resident(ctx, W):
    """urh_spectrogram_bgra_stream at the decimal and reversed ranges gives the resident images byte for byte: the segments of
    create_image_segments in pieces and in groups, and one transposed image"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    x = _segment_capture(W)
    spec = Spectrogram(x, W, 0.5)
    segments = [(s, e - s) for s, e, _ in spec.segment_bounds()]
    seg_len = segments[0][1]
    for L in (65536, 65537):
        for lo, hi in DECIMAL_RANGES[:2] + REVERSED_RANGES[:1]:
            spec.data_min, spec.data_max = lo, hi
            ref = list(spec.create_image_segments(colormap=CMAPS[L]))
            for chunk in (seg_len // 3, 3 * seg_len):
                got = _stream_images(ctx, spec, x, segments, False, CMAPS[L], chunk)
                assert len(got) == len(ref) and all(_same_bytes(a, b) for a, b in zip(got, ref)), (W, L, lo, hi, chunk)
            ref_t = spec.create_spectrogram_image(transpose=True, colormap=CMAPS[L])
            (got_t,) = _stream_images(ctx, spec, x, [(0, len(x))], True, CMAPS[L], seg_len // 2)
            assert _same_bytes(got_t, ref_t), (W, L, lo, hi)


# ---- capture conversions (k_convert) ------------------------------------------------------------------------------------------------
def _float_sources():
    """float32 samples where the conversions go wrong: NaN payloads, +-inf, +-0, subnormals, +-1 and their neighbours, values
    past +-1 that wrap the target, products at and past 2^31 (numpy's int32 step gives INT_MIN, low bits 0), and every truncation
    boundary k / scale - offset of each target with the float32 values 1 and 2 ulp to either side"""
    f32 = np.float32
    nan = np.array([0x7FC00000, 0x7F800001, 0x7FBFFFFF, 0xFFC00000, 0xFFC00001, 0x7FFFFFFF, 0xFFFFFFFF], np.uint32).view(f32)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38, 1.0, -1.0, 200.0,
                        -200.0, 1.5, -1.5, 2.0, -2.0, 3.0, -3.0, 258.0, -258.0, 1000.0, -1000.0, 65536.0, -65536.0, 3e9, -3e9, 1e10,
                        -1e10, 1e30, -1e30, 3.4028235e38, -3.4028235e38], f32)
    edges = [nan, special]
    for scale, offset, ks in ((127, 0, np.arange(-400, 401)), (127, 1, np.arange(-400, 801)),
                              (32767, 0, np.arange(-70000, 70001)), (32767, 1, np.arange(-70000, 140001, 3))):
        big = np.array([2.0 ** 31, -(2.0 ** 31), 2.0 ** 32, 2.0 ** 24, -(2.0 ** 24)])
        t = np.concatenate([ks / scale, big / scale]) - offset
        t = t.astype(f32)
        up, down = t, t
        edges.append(t)
        for _ in range(2):
            up, down = np.nextafter(up, f32(np.inf)), np.nextafter(down, f32(-np.inf))
            edges += [up, down]
    v = np.concatenate(edges)
    return np.resize(v, (len(v) + 1) // 2 * 2).reshape(-1, 2)


def _int_sources(dtype):
    """every value of an integer dtype, as samples"""
    info = np.iinfo(dtype)
    return np.arange(info.min, info.max + 1).astype(dtype).reshape(-1, 2)


def _sources(src):
    return _float_sources() if src == np.float32 else _int_sources(src)


def _device_convert(ctx, d_in, src, dst, count, out=None):
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray

    out = DeviceArray(ctx, (count,), dst) if out is None else out
    ctx.check(ctx.lib.urh_convert_iq(ctx.handle, C.c_void_p(d_in), _lib.dtype_code(src), C.c_void_p(out.ptr), _lib.dtype_code(dst),
                                     count))
    return out


def test_conversion_literals(oracle):
    """numpy on x86-64 wraps 200 x 127 into int8 56 and sends NaN, inf and 1e10 to 0 in every integer target; the device does too.
    Should numpy on some host differ, this fails instead of agreeing with another specification."""
    from urh_b200.signalprocessing.IQArray import IQArray

    x = np.array([[200.0, np.nan], [np.inf, 1e10]], np.float32)
    want = {np.int8: [[56, 0], [0, 0]]}
    for dst in INT_TYPES:
        with np.errstate(all="ignore"):
            ref = oracle.convert_iq(x, dst)
        assert np.array_equal(ref[:, 1], [0, 0]) and ref[1, 0] == 0, dst
        if dst in want:
            assert np.array_equal(ref, want[dst])
        assert _same_bytes(IQArray(x.copy()).convert_to(dst), ref), dst


@pytest.mark.parametrize("src", ALL_TYPES)
@pytest.mark.parametrize("dst", ALL_TYPES)
def test_conversion_every_edge(oracle, src, dst):
    """IQArray.convert_to == the reference's numpy expression (oracle.convert_iq) byte for byte: every integer source value, the
    float32 edge values; also one sample alone"""
    from urh_b200.signalprocessing.IQArray import IQArray

    x = _sources(src)
    with np.errstate(all="ignore"):
        want = oracle.convert_iq(x, dst)
    got = IQArray(x.copy()).convert_to(dst)
    bad = np.flatnonzero(np.ascontiguousarray(got).view(np.uint8) != np.ascontiguousarray(want).view(np.uint8))
    assert _same_bytes(got, want), (src, dst, len(bad), x.reshape(-1)[bad[:4] // np.dtype(dst).itemsize])
    for i in (0, len(x) // 2, len(x) - 1):
        assert _same_bytes(IQArray(x[i:i + 1].copy()).convert_to(dst), want[i:i + 1]), (src, dst, i)


@pytest.mark.parametrize("src", ALL_TYPES)
def test_conversion_counts_offsets_and_stream(ctx, oracle, sm_count, src):
    """urh_convert_iq on an odd element count (the element after it untouched), on device views starting at sample 1 and 3, over
    more than sm_count x 32 x 256 elements (the grid-stride loop runs again), and urh_convert_iq_stream on the same samples"""
    from urh_b200 import _lib
    from urh_b200.device import to_device

    base = _sources(src)
    n = -(-(2 * sm_count * 32 * 256 + 7) // 2)
    x = np.ascontiguousarray(np.resize(base, (n, 2)))
    d_x = to_device(x, ctx)
    for dst in ALL_TYPES:
        if dst == src:
            continue
        with np.errstate(all="ignore"):
            want = oracle.convert_iq(x, dst)
        got = _device_convert(ctx, d_x.ptr, src, dst, 2 * n).get().reshape(n, 2)
        assert _same_bytes(got, want), (src, dst, "grid-stride")
        count = 2 * 1001 + 1
        out = to_device(np.full((count + 1) * np.dtype(dst).itemsize, 0xA5, np.uint8).view(dst), ctx)
        got = _device_convert(ctx, d_x.ptr, src, dst, count, out).get()
        assert _same_bytes(got[:count], want.reshape(-1)[:count]), (src, dst, "odd count")
        assert np.all(got[count:].view(np.uint8) == 0xA5), (src, dst, "wrote past the count")
        for off in (1, 3):
            view = d_x[off:]
            got = _device_convert(ctx, view.ptr, src, dst, 2 * (n - off)).get().reshape(-1, 2)
            assert _same_bytes(got, want[off:]), (src, dst, off)
        small = np.ascontiguousarray(x[: len(base)])
        d_small = to_device(small, ctx)
        ref = _device_convert(ctx, d_small.ptr, src, dst, small.size).get().reshape(-1, 2)
        for chunk in (4099, 1 << 16):
            out = np.empty_like(ref)
            ctx.check(ctx.lib.urh_convert_iq_stream(ctx.handle, _ptr(small), _lib.dtype_code(src), _ptr(out), _lib.dtype_code(dst),
                                                    len(small), chunk, 2))
            assert _same_bytes(out, ref), (src, dst, chunk)


# ---- the strided sample gather (urh_gather_samples) ----------------------------------------------------------------------------------
def _slices(n):
    return [(None, None, -1), (None, None, 2), (n + 5, None, -2), (-n - 5, None, 3), (-n - 5, n + 5, 7), (n + 5, -n - 5, -7),
            (None, None, n - 1), (None, None, -(n - 1)), (n - 1, 0, -(n - 1)), (3, None, n + 3), (None, None, -(n + 3)),
            (5, 3, 2), (3, 5, -2), (n + 5, n + 10, 3), (-n - 10, -n - 5, -3), (10, 400, -1), (400, 10, -1), (400, 10, -13)]


def test_gather_against_numpy_slicing(ctx):
    """urh_gather_samples == x[start:stop:step] for positive and negative steps, starts and stops past either end, empty results
    and steps of +-1, +-(n - 1) and beyond"""
    from urh_b200.device import DeviceArray, to_device

    n = 1000
    rng = np.random.default_rng(11)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    d_x = to_device(x.view(np.float32).reshape(-1, 2), ctx)
    for args in _slices(n):
        want = x[slice(*args)]
        start, stop, step = slice(*args).indices(n)
        count = len(range(start, stop, step))
        assert count == len(want)
        out = DeviceArray(ctx, (count + 1, 2), np.float32).zero()
        ctx.check(ctx.lib.urh_gather_samples(ctx.handle, C.c_void_p(d_x.ptr), n, start, step, count, C.c_void_p(out.ptr)))
        got = out.get()
        assert _same_bytes(got[:count].reshape(-1).view(np.complex64), want), args
        assert np.all(got[count] == 0), args


def test_image_of_device_slice_equals_host_slice(ctx):
    """create_spectrogram_image(start, stop, step) on device samples == the image of the numpy slice of the host samples"""
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n, W = 1000, 128
    x = _capture(n, W, seed=5)
    d_x = to_device(x, ctx)
    cmap = CMAPS[1025]
    for args in _slices(n) + [(None, -1, None), (1, None, -1)]:
        want = Spectrogram(x[slice(*args)], W).create_spectrogram_image(colormap=cmap)
        got = Spectrogram(d_x, W).create_spectrogram_image(*args, colormap=cmap)
        assert got.shape == want.shape and np.array_equal(got.get(), want), args
