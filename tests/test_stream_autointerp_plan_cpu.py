"""CPU: the plans and footprints of the streamed auto-interpretation entries, without a device: the noise-chunk windows
(urh_stream_windows with URH_FILTER_NOISE), the conversion windows (URH_FILTER_CONVERT), the footprints of the streamed noise level,
conversion and segmentation, and the decision of estimate() between its resident and its host path."""
import ctypes as C

import numpy as np
import pytest

SLICES = 64


@pytest.fixture(scope="module")
def L():
    from urh_b200 import _lib, build

    build.build()
    return _lib


def windows(L, entry, n, out_len, p0, p1, cs):
    lib = L.load_library()
    count = C.c_int64(0)
    args = (entry, n, out_len, p0, p1, cs, None, None, 0)
    assert lib.urh_stream_windows(*args, None, 0, C.byref(count)) == 0
    w = np.zeros((max(count.value, 1), 4), np.int64)
    assert lib.urh_stream_windows(*args, w.ctypes.data_as(C.c_void_p), count.value, C.byref(count)) == 0
    return w[: count.value]


def chunking(n):
    """AutoInterpretation._chunking"""
    chunksize = max(1, int(n * 1 / 100))
    return chunksize, n // chunksize


def slices_in_sample_order(n, cs, nchunks):
    """[s0, s1) of every slice of every noise chunk as k_chunk_partial reduces it, in ascending sample order"""
    per = -(-cs // SLICES)
    out = []
    for j in range(nchunks - 1, -1, -1):
        c0 = n - (j + 1) * cs
        for sl in range(SLICES):
            s0 = min(c0 + sl * per, c0 + cs)
            out.append((s0, min(s0 + per, c0 + cs)))
    return out


def check_noise_plan(L, n, cs, nchunks, chunk):
    w = windows(L, L.FILTER_NOISE, n, 0, cs, nchunks, chunk)
    sl = slices_in_sample_order(n, cs, nchunks)
    per = -(-cs // SLICES)
    # every slice lies in exactly one window, in order
    assert w[0, 0] == 0 and w[-1, 1] == len(sl)
    assert np.array_equal(w[1:, 0], w[:-1, 1])
    assert (w[:, 1] > w[:, 0]).all()
    head = n - nchunks * cs
    for k0, k1, a, b in w:
        assert a == sl[k0][0] and b == sl[k1 - 1][1]   # the window is exactly its slices' samples
        assert all(sl[g][0] >= a and sl[g][1] <= b for g in range(k0, k1))
        assert b - a <= max(chunk, per)
        assert a >= head   # the head before the first noise chunk is never uploaded
    assert (np.diff(w[:, 2]) >= 0).all() and (np.diff(w[:, 3]) >= 0).all()   # windows ascend
    assert np.array_equal(w[1:, 2], w[:-1, 3])   # and leave no sample between them
    return w


@pytest.mark.parametrize("n", [4, 5, 63, 64, 99, 100, 101, 199, 640, 6399, 6400, 6401, 10_007, 123_457, 1_000_003])
@pytest.mark.parametrize("chunk", [1, 7, 64, 1000, 1 << 14])
def test_noise_windows_autointerp_chunking(L, n, chunk):
    cs, nchunks = chunking(n)
    check_noise_plan(L, n, cs, nchunks, chunk)


@pytest.mark.parametrize("n, cs, nchunks", [(10, 1, 3), (1000, 10, 100), (10_000, 33, 300), (70_000, 700, 100), (12_345, 123, 100)])
@pytest.mark.parametrize("chunk", [1, 5, 11, 64, 512, 1 << 20])
def test_noise_windows_any_chunking(L, n, cs, nchunks, chunk):
    check_noise_plan(L, n, cs, nchunks, chunk)


def test_noise_window_of_one_long_slice(L):
    # a slice longer than a chunk is a window of its own
    n, cs, nchunks = 640_123, 6400, 100
    w = check_noise_plan(L, n, cs, nchunks, 50)
    assert len(w) == nchunks * SLICES and (w[:, 1] - w[:, 0] == 1).all()
    assert ((w[:, 3] - w[:, 2]) == 100).all()


def test_noise_windows_reject_bad_chunking(L):
    lib = L.load_library()
    count = C.c_int64(0)
    for cs, nchunks in [(0, 10), (10, 0), (11, 10)]:
        assert lib.urh_stream_windows(L.FILTER_NOISE, 100, 0, cs, nchunks, 1000, None, None, 0, None, 0, C.byref(count)) != 0


@pytest.mark.parametrize("n", [1, 999, 1000, 1001, 12_345])
@pytest.mark.parametrize("chunk", [1, 1000, 4096])
def test_convert_windows_cover_once(L, n, chunk):
    w = windows(L, L.FILTER_CONVERT, n, n, L.DT_I8, 0, chunk)
    assert w[0, 0] == 0 and w[-1, 1] == n
    assert np.array_equal(w[1:, 0], w[:-1, 1])
    assert np.array_equal(w[:, :2], w[:, 2:]) and ((w[:, 1] - w[:, 0]) <= chunk).all()


# ---- footprints ------------------------------------------------------------------------------------------------------------------------
DTYPES = [np.int8, np.uint8, np.int16, np.uint16, np.float32]


@pytest.mark.parametrize("dtype", DTYPES)
def test_streamed_footprints_are_flat_in_n(L, dtype):
    from urh_b200.cythonext import signal_functions as sf

    noise, convert, seg = set(), set(), set()
    for n in [1 << 26, 1 << 28, 1 << 31, 1 << 34, 1 << 36]:
        cs, nchunks = chunking(n)
        noise.add(sf.filter_footprint(L.FILTER_NOISE, n, 0, dtype, cs, nchunks))
        convert.add(sf.filter_footprint(L.FILTER_CONVERT, n, n, dtype, L.DT_F32, 0))
        seg.add(sf.stream_footprint(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES))
    assert len(noise) == 1 and len(convert) == 1 and len(seg) == 1
    # and far below the resident forms at those sizes
    n = 1 << 34
    cs, nchunks = chunking(n)
    assert sf.filter_footprint(L.FILTER_NOISE, n, 0, dtype, cs, nchunks, resident=True) > 10 * noise.pop()
    assert sf.stream_footprint(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES | L.STREAM_RESIDENT) > 10 * seg.pop()


def test_resident_footprints_grow_with_the_capture(L):
    from urh_b200.cythonext import signal_functions as sf

    for dtype in DTYPES:
        ib = 2 * np.dtype(dtype).itemsize
        n = 1 << 30
        cs, nchunks = chunking(n)
        assert sf.filter_footprint(L.FILTER_NOISE, n, 0, dtype, cs, nchunks, resident=True) >= n * ib
        assert sf.filter_footprint(L.FILTER_CONVERT, n, n, dtype, L.DT_I16, 0, resident=True) >= n * (ib + 4)
        assert sf.stream_footprint(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES | L.STREAM_RESIDENT) >= n * (ib + 8)


def test_footprint_rejects_a_streamed_estimate(L):
    out = C.c_int64(0)
    lib = L.load_library()
    assert lib.urh_stream_footprint(1000, L.DT_F32, 0, 0, 2, L.STREAM_ESTIMATE, -1, C.byref(out)) != 0
    assert lib.urh_stream_footprint(1000, L.DT_F32, 0, 0, 2, L.STREAM_ESTIMATE | L.STREAM_RESIDENT, -1, C.byref(out)) == 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_estimate_decision_is_the_c_formula(L, dtype):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.cythonext import signal_functions as sf

    for n in [1000, 1 << 20, 1 << 30, 1 << 33]:
        ib = 2 * np.dtype(dtype).itemsize
        resident = sf.stream_footprint(n, dtype, 0, L.STREAM_ESTIMATE | L.STREAM_RESIDENT)
        psk = sf.stream_footprint(n, dtype, 0, L.STREAM_AFP_DEMOD | L.STREAM_PSK | L.STREAM_RESIDENT)
        assert resident >= psk + 8 * n and psk >= n * (ib + 4)   # capture, magnitudes, qad and the Costas tables
        for mod in (L.STREAM_AFP_DEMOD, L.STREAM_AFP_DEMOD | L.STREAM_PSK4):
            if mod & L.STREAM_PSK4:
                continue
            assert resident >= sf.stream_footprint(n, dtype, 0, mod | L.STREAM_RESIDENT) + 8 * n
        for budget in (resident - 1, resident, resident + 1):
            assert AI.estimate_streams(n, dtype, budget) == (resident > budget)


@pytest.mark.parametrize("dtype", DTYPES)
def test_switch_happens_at_the_budget(L, dtype):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.cythonext import signal_functions as sf

    n = 5_000_000
    cs, nchunks = chunking(n)
    r_noise = sf.filter_footprint(L.FILTER_NOISE, n, 0, dtype, cs, nchunks, resident=True)
    assert AI.noise_level_streams(n, dtype, r_noise - 1) and not AI.noise_level_streams(n, dtype, r_noise)
    assert not AI.noise_level_streams(3, dtype, 0)   # three samples or fewer: no noise level, nothing to stream
    r_conv = sf.filter_footprint(L.FILTER_CONVERT, n, n, dtype, L.DT_I8, 0, resident=True)
    assert sf.filter_use_stream(L.FILTER_CONVERT, n, n, dtype, L.DT_I8, 0, r_conv - 1)
    assert not sf.filter_use_stream(L.FILTER_CONVERT, n, n, dtype, L.DT_I8, 0, r_conv)
    r_seg = sf.stream_footprint(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES | L.STREAM_RESIDENT)
    assert sf.use_stream(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES, r_seg - 1)
    assert not sf.use_stream(n, dtype, 0, L.STREAM_SEGMENT_MESSAGES, r_seg)
