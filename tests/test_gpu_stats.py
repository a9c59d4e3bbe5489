"""GPU parity: auto-interpretation statistics (stats.cu + urh_b200.ainterpretation) vs golden vectors / oracle."""
import numpy as np
import pytest

from conftest import CAPTURES, bits_equal, load_golden, synth_fsk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def AI():
    from urh_b200.ainterpretation import AutoInterpretation

    return AutoInterpretation


@pytest.mark.parametrize("name", CAPTURES)
def test_magnitudes_noise_segments_golden(AI, oracle, name):
    from urh_b200.cythonext import util

    g = load_golden("capture_" + name)
    mags = util.get_magnitudes(g["iq"])
    assert mags.dtype == np.float64
    assert np.array_equal(mags, oracle.get_magnitudes(g["iq"]), equal_nan=True)
    assert np.array_equal(mags[:64], g["mag_head"])
    assert AI.detect_noise_level(mags) == float(g["auto_noise"])
    assert AI.detect_noise_level_iq(g["iq"]) == float(g["auto_noise"])
    seg = AI.segment_messages_from_magnitudes(mags, float(g["noise"]))
    assert np.array_equal(np.array(seg, dtype=np.int64).reshape(-1, 2), g["segments"])
    seg32 = AI.segment_messages_from_magnitudes(mags.astype(np.float32), float(g["noise"]))
    assert seg32 == oracle.segment_messages_from_magnitudes(mags.astype(np.float32), float(g["noise"]))


@pytest.mark.parametrize("name", CAPTURES)
def test_detect_center_golden(AI, name):
    g = load_golden("capture_" + name)
    m = g["meta"]
    c = AI.detect_center(g["qad_" + m["mod"]])
    gc = float(g["detect_center"])
    if np.isnan(gc):
        assert c is None
    else:
        # variance accumulated in double on the GPU vs numpy's pairwise float32 (DESIGN.md): bin edges move by
        # ~1e-7 relative, so the center (mean of two bin edges) agrees to ~1e-6 of the signal scale
        assert c is not None and abs(c - gc) <= 2e-6 * max(1.0, abs(gc)), (c, gc)


def test_segmentation_randomised(AI, oracle):
    rng = np.random.default_rng(3)
    for trial in range(40):
        n = int(rng.choice([1, 9, 10, 11, 100, 2047, 2048, 2049, 30000]))
        period = int(rng.integers(5, 400))
        env = np.repeat(rng.integers(0, 2, n // period + 1), period)[:n].astype(np.float64)
        mags = env + 0.3 * rng.random(n)
        flips = rng.random(n) < 0.03
        mags[flips] = 1.3 - mags[flips]
        for arr in (mags, mags.astype(np.float32)):
            assert AI.segment_messages_from_magnitudes(arr, 0.65) == oracle.segment_messages_from_magnitudes(arr, 0.65), (trial, n)


def test_plateaus_median_decibel(AI, oracle):
    from urh_b200.cythonext import auto_interpretation as cai
    from urh_b200.cythonext import util

    rng = np.random.default_rng(5)
    for n in (1, 7, 100, 5000, 70000):
        period = int(rng.integers(3, 50))
        x = (np.repeat(rng.standard_normal(n // period + 1), period)[:n] + 0.05 * rng.standard_normal(n)).astype(np.float32)
        for pct in (25, 100, 3):
            assert np.array_equal(cai.get_plateau_lengths(x, 0.1, pct), oracle.get_plateau_lengths(x, 0.1, pct)), (n, pct)
        d = rng.standard_normal(n)
        for k in (3, 11, 4):
            assert np.array_equal(cai.median_filter(d, k), oracle.median_filter(d, k)), (n, k)
    z = (rng.standard_normal((37, 64)) + 1j * rng.standard_normal((37, 64))).astype(np.complex64)
    db = util.arr2decibel(z)
    ref = oracle.arr2decibel(z)
    assert db.shape == ref.shape and db.dtype == np.float32
    assert np.max(np.abs(db - ref)) <= 1e-5  # CUDA log10f vs glibc log10f: <= 2 ulp


def test_detect_center_large_vs_oracle(AI, oracle):
    from urh_b200.cythonext import signal_functions as sf

    iq = synth_fsk(400000, sps=100, seed=2, gap_every=50000)
    qad = sf.afp_demod(iq, 0.05, "FSK", 2)
    c = AI.detect_center(qad)
    ref = oracle.detect_center(qad)
    assert abs(c - ref) <= 2e-6
    c2 = AI.detect_center(qad, max_size=50000)
    assert abs(c2 - oracle.detect_center(qad, max_size=50000)) <= 2e-6


def test_estimate_matches_golden(AI):
    for name in ("fsk", "ask", "enocean", "homematic"):
        g = load_golden("capture_" + name)
        est = g["meta"]["estimate"]
        res = AI.estimate(g["iq"])
        assert (res is None) == (est is None)
        if est is not None:
            assert res["modulation_type"] == est["modulation_type"]
            assert res["bit_length"] == est["bit_length"]
            assert res["tolerance"] == est["tolerance"]
            assert res["noise"] == est["noise"]
            assert abs(res["center"] - est["center"]) <= 1e-5 * max(1.0, abs(est["center"]))


# ---- demod + detect_center from one pass ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CAPTURES)
def test_demod_detect_center_matches_two_step_golden(AI, name):
    """urh_afp_demod_stats + urh_center_histogram_tiles == afp_demod followed by detect_center (golden from the reference)."""
    g = load_golden("capture_" + name)
    m = g["meta"]
    mod = m["mod"]
    if mod not in ("ASK", "FSK"):
        pytest.skip("ASK/FSK only")
    qad, center = AI.demod_detect_center(g["iq"], float(g["noise"]), mod)
    assert bits_equal(qad.get(), g["qad_" + mod]) == 0
    two_step = AI.detect_center(g["qad_" + mod])
    assert (center is None) == (two_step is None)
    gc = float(g["detect_center"])
    if center is not None:
        # the stand-alone detect_center replays numpy's float32 variance bit for bit; the fused pass takes the variance from the
        # demodulator's double tile sums (no extra pass): the bin width moves by ~1e-7 relative, the center within 2e-6
        assert float(two_step) == gc
        assert abs(center - gc) <= 2e-6 * max(1.0, abs(gc))
        _, exact = AI.demod_detect_center(g["iq"], float(g["noise"]), mod, bitwise=True)
        assert float(exact) == gc


@pytest.mark.parametrize("n", [3, 2047, 2048, 2049, 70001, 1 << 20, 2 * 4096 * 2048 + 4097])
@pytest.mark.parametrize("max_size", [None, 5000])
def test_demod_detect_center_sizes(AI, n, max_size):
    from urh_b200.cythonext import signal_functions as sf
    iq = synth_fsk(n, seed=n)
    qad, center = AI.demod_detect_center(iq, 0.05, "FSK", max_size)
    ref_qad = sf.afp_demod(iq, 0.05, "FSK", 2)
    assert bits_equal(qad.get(), ref_qad) == 0
    two_step = AI.detect_center(ref_qad, max_size)
    assert (center is None) == (two_step is None)
    if center is not None:
        assert abs(center - two_step) <= 2e-6 * max(1.0, abs(two_step))
        _, exact = AI.demod_detect_center(iq, 0.05, "FSK", max_size, bitwise=True)
        assert float(exact) == float(two_step)


def test_demod_center_digitize_matches_three_calls(AI):
    from urh_b200.cythonext import signal_functions as sf
    iq = synth_fsk(1 << 20, seed=5)
    center, rows = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100)
    qad = sf.afp_demod(iq, 0.05, "FSK", 2)
    c2 = AI.detect_center(qad)
    assert abs(center - c2) <= 2e-6
    c2 = center
    assert np.array_equal(rows, sf.grab_pulse_lens(qad, c2, 5, "FSK", 100))
    assert rows[:, 1].sum() == len(iq) - 5


@pytest.mark.parametrize("nbins_target", [7, 64, 1500, 7000, 20000])
def test_tile_histogram_counts_equal_numpy(AI, nbins_target):
    """urh_center_histogram_tiles (float edge thresholds, register-counted hot bins) == np.histogram on the same edges."""
    import ctypes as C
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device
    n = 300_001
    iq = synth_fsk(n, seed=nbins_target, gap_every=50_000)
    ctx = _lib.default_context()
    d_iq = to_device(iq, ctx)
    qad = DeviceArray(ctx, (n,), np.float32)
    kept = C.c_int64(0)
    ctx.check(ctx.lib.urh_afp_demod_tiles(ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(d_iq.dtype), n, 0.05, _lib.MOD_FSK,
                                          C.c_void_p(qad.ptr), 0, C.byref(kept)))
    host = qad.get()
    rect_all = host[host > -4]
    assert kept.value == len(rect_all)
    r0, r1 = AI.center_rank_window(kept.value)
    rect = rect_all[r0:r1]
    w = np.zeros(5)
    ctx.check(ctx.lib.urh_center_window_stats(ctx.handle, C.c_void_p(qad.ptr), n, r0, r1, w.ctypes.data_as(C.c_void_p)))
    assert int(w[0]) == len(rect) and np.float32(w[1]) == rect.min() and np.float32(w[2]) == rect.max()
    assert abs(w[3] - rect.astype(np.float64).sum()) <= 1e-9 * len(rect)
    # edges that cut through the data: interior start/stop so that out-of-range samples exist on both sides
    lo, hi = float(np.percentile(rect, 1)), float(np.percentile(rect, 99.5))
    step = (hi - lo) / nbins_target
    edges = np.arange(lo, hi + step, step)
    nbins = len(edges) - 1
    y = np.zeros(nbins, dtype=np.int64)
    ctx.check(ctx.lib.urh_center_histogram_tiles(ctx.handle, C.c_void_p(qad.ptr), n, r0, r1, C.c_double(edges[0]),
                                                 C.c_double(edges[1] - edges[0]), nbins, y.ctypes.data_as(C.c_void_p)))
    # np.arange fills start + i*delta: rebuild exactly those edges for numpy
    exact_edges = edges[0] + np.arange(nbins + 1) * (edges[1] - edges[0])
    ref, _ = np.histogram(rect, bins=exact_edges)
    assert np.array_equal(y, ref)
    y2 = np.zeros(nbins, dtype=np.int64)
    ctx.check(ctx.lib.urh_center_histogram(ctx.handle, C.c_void_p(qad.ptr), n, r0, r1, C.c_double(edges[0]),
                                           C.c_double(edges[1] - edges[0]), nbins, y2.ctypes.data_as(C.c_void_p)))
    assert np.array_equal(y2, ref)


# ---- np.var replayed bit for bit (pairwise.cu) -> detect_center bit-identical ------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 9, 127, 128, 129, 300, 2047, 2049, 70_001, 1_000_003, 5_000_000])
def test_window_var_is_numpys_bit_for_bit(n):
    """urh_center_stats: {mean, var} of the rank-trimmed window == np.mean / np.var of the same float32 array, every bit"""
    import ctypes as C
    from urh_b200 import _lib
    from urh_b200.device import to_device
    rng = np.random.default_rng(n)
    x = (rng.standard_normal(n) * 0.3 + rng.choice([-0.3, 0.3], n)).astype(np.float32)
    x[rng.random(n) < 0.2] = -4.0   # noise sentinel: not kept
    ctx = _lib.default_context()
    d = to_device(x, ctx)
    st = np.zeros(7)
    ctx.check(ctx.lib.urh_center_stats(ctx.handle, C.c_void_p(d.ptr), n, -1, st.ctypes.data_as(C.c_void_p)))
    rect = x[x > -4]
    rect = rect[int(0.05 * len(rect)):int(0.95 * len(rect))]
    assert int(st[0]) == int((x > -4).sum())
    if len(rect) == 0:
        return
    assert np.float32(st[5]).view(np.uint32) == np.float32(np.mean(rect)).view(np.uint32)
    assert np.float32(st[6]).view(np.uint32) == np.float32(np.var(rect)).view(np.uint32)


@pytest.mark.parametrize("name", CAPTURES)
def test_detect_center_bit_identical_golden(AI, oracle, name):
    g = load_golden("capture_" + name)
    mod = g["meta"]["mod"]
    qad = g["qad_" + mod]
    mine = AI.detect_center(qad)
    ref = oracle.detect_center(qad)
    assert (mine is None) == (ref is None)
    if mine is not None:
        assert float(mine) == float(ref) == float(g["detect_center"])


def test_detect_center_bit_identical_random(AI, oracle):
    rng = np.random.default_rng(77)
    for trial in range(40):
        n = int(rng.integers(50, 400_000))
        lv = rng.uniform(-2, 2, 2)
        x = (np.repeat(rng.choice(lv, n // 50 + 1), 50)[:n] + rng.standard_normal(n) * rng.uniform(0.005, 0.2)).astype(np.float32)
        x[rng.random(n) < rng.uniform(0, 0.5)] = -4.0
        mine, ref = AI.detect_center(x), oracle.detect_center(x)
        assert (mine is None) == (ref is None), trial
        if mine is not None:
            assert float(mine) == float(ref), (trial, n, mine, ref)


def test_demod_detect_center_bitwise_option(AI, oracle):
    iq = synth_fsk(1_500_000, seed=21, gap_every=100_000)
    qad, c = AI.demod_detect_center(iq, 0.05, "FSK", bitwise=True)
    assert float(c) == float(oracle.detect_center(qad.get()))
