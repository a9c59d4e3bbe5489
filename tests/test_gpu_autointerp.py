"""GPU: the auto-interpretation kernels (stats.cu, pairwise.cu, modulation.cu) against the reference's recorded answers
(tests/golden/ref_autointerp.json, see tests/test_autointerp_reference_cpu.py) and the oracle, on the case matrix of
tests/autointerp_cases.py: every IQ dtype, sizes around the chunk, tile and power-of-two edges, values on the decision
thresholds, NaN / inf / subnormal samples.  Bit-exact wherever the reference's arithmetic is replayed; the wavelet features,
whose float32 FFT rounds differently from pocketfft, are held to a float64 truth instead."""
import ctypes as C

import numpy as np
import pytest

import autointerp_cases as cases
from oracle.cassette import digest, fingerprint, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def AI():
    from urh_b200.ainterpretation import AutoInterpretation
    return AutoInterpretation


def outcome(thunk):
    try:
        return thunk()
    except Exception as e:   # noqa: BLE001 -- the exception is the answer
        return ("raises", type(e).__name__)


def dev(a):
    from urh_b200.device import to_device
    return to_device(np.ascontiguousarray(a))


# ---- magnitudes -----------------------------------------------------------------------------------------------------------
def test_magnitudes_bit_exact(oracle):
    from urh_b200.cythonext import util
    want = cases.recorded("test_magnitudes_pinned")
    for i, iq in enumerate(cases.magnitude_cases()):
        got = util.get_magnitudes(iq)
        assert got.dtype == np.float64 and got.shape == (len(iq),)
        assert digest(cases.canon(got)) == want[i], (iq.dtype, len(iq))
        assert np.array_equal(got, oracle.get_magnitudes(iq), equal_nan=True), (iq.dtype, len(iq))
        if len(iq) == 257:   # DeviceArray in, DeviceArray out
            d = util.get_magnitudes(dev(iq))
            assert digest(cases.canon(d.get())) == want[i]


def test_magnitudes_extremes_explicit():
    """the values the matrix plants, spelled out: int16 (-32768, -32768) wraps to a negative int32 sum of squares"""
    from urh_b200.cythonext import util
    got = util.get_magnitudes(np.array([[-32768, -32768], [-128, -128]], np.int16))
    assert np.isnan(got[0]) and got[1] == np.sqrt(2 * 128 * 128)
    assert np.isnan(util.get_magnitudes(np.array([[65535, 65535]], np.uint16))[0])   # 2 * 65535^2 wraps negative as well
    f = util.get_magnitudes(np.array([[1e20, 1e20], [1e-45, 1e-45], [np.inf, np.nan]], np.float32))
    assert f[0] == np.inf and f[1] == np.float64(np.sqrt(np.float32(0))) and np.isnan(f[2])


# ---- noise level ----------------------------------------------------------------------------------------------------------
def test_noise_level_host_and_device(AI):
    want = cases.recorded("test_noise_level_pinned")
    for i, (name, mags) in enumerate(cases.noise_cases()):
        assert outcome(lambda: AI.detect_noise_level(mags)) == want[i], name
        assert outcome(lambda: AI.detect_noise_level(dev(mags))) == want[i], name


def test_noise_level_float32_chunk_means_are_numpys(AI):
    """np.mean of a float32 chunk is numpy's float32 pairwise sum: a double sum puts this chunk on the quiet edge (0.0209)"""
    mags = cases.edge_f32_noise()
    assert AI.detect_noise_level(mags) == 0.01
    # float64 magnitudes of the same values: np.mean sums in double, the rounded mean lies on the edge, the chunk is quiet
    assert AI.detect_noise_level(mags.astype(np.float64)) == AI.detect_noise_level(dev(mags.astype(np.float64))) == 0.0211


def test_noise_level_iq_every_dtype(AI):
    want = cases.recorded("test_noise_level_iq_pinned")
    for i, (name, iq) in enumerate(cases.noise_iq_cases()):
        assert outcome(lambda: AI.detect_noise_level_iq(iq)) == want[i], name
        assert outcome(lambda: AI.detect_noise_level_iq(dev(iq))) == want[i], name


# ---- segmentation ---------------------------------------------------------------------------------------------------------
def test_segments(AI, oracle):
    want = cases.recorded("test_segments_pinned")
    for i, (name, mags, thr) in enumerate(cases.segment_cases()):
        got = AI.segment_messages_from_magnitudes(mags, thr)
        assert fingerprint(got) == want[i], name
        if name.startswith("70000_messages"):
            assert len(got) == 70_000


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_segments_device_slices_at_odd_offsets(AI, oracle, dtype):
    """DeviceArray views that start off the vector alignment take the scalar load path of the dense pass"""
    rng = np.random.default_rng(9)
    n = 3 * cases.TILE + 50
    a = np.repeat(rng.integers(0, 2, n // 7 + 1), rng.integers(6, 14))[:n].astype(dtype)
    a[rng.random(n) < 0.02] = cases.SEG_THR
    d = dev(a)
    for off in (1, 2, 3, 5, 7):
        for end in (n, n - 3):
            got = AI.segment_messages_from_magnitudes(d[off:end], cases.SEG_THR)
            assert got == oracle.segment_messages_from_magnitudes(a[off:end], cases.SEG_THR), (off, end)


# ---- plateau lengths, median filter, arr2decibel ----------------------------------------------------------------------------
def test_plateau_lengths():
    from urh_b200.cythonext import auto_interpretation as cai
    want = cases.recorded("test_plateau_lengths_pinned")
    for i, (name, rect, center, pct) in enumerate(cases.plateau_cases()):
        got = cai.get_plateau_lengths(rect, center, pct)
        assert got.dtype == np.uint64 and same(got, want[i]), name


def test_median_filter():
    from urh_b200.cythonext import auto_interpretation as cai
    want = cases.recorded("test_median_filter_pinned")
    for i, (name, data, k) in enumerate(cases.median_cases()):
        got = cai.median_filter(data, k)
        assert got.dtype == np.float32 and same(got, want[i]), name
        assert np.array_equal(np.signbit(got), np.signbit(np.asarray(cai.median_filter(dev(data), k).get()))), name
    with pytest.raises(Exception, match="k must be in 1..64"):
        cai.median_filter(np.ones(100), 65)


def test_arr2decibel_ulps(oracle):
    """10 log10(re^2 + im^2) in float32: CUDA log10f within 2 ulp of glibc's; exactly -inf for 0"""
    from urh_b200.cythonext import util
    rng = np.random.default_rng(11)
    z = (rng.standard_normal((97, 64)) * np.exp(rng.uniform(-40, 40, (97, 64))) + 1j * rng.standard_normal((97, 64))).astype(np.complex64)
    special = np.array([0, -0.0, np.inf, complex(0, -np.inf), complex(np.nan, 0), complex(1e-45, 0), complex(1e-42, 1e-41),
                        complex(1e-20, 0), complex(3e38, 3e38), 1, 1j], dtype=np.complex64)
    z[0, :len(special)] = special
    got, ref = util.arr2decibel(z), oracle.arr2decibel(z)
    assert got.shape == ref.shape and got.dtype == np.float32
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)])
    assert got[0, 0] == -np.inf and got[0, 1] == -np.inf and got[0, 2] == np.inf
    ulp = np.abs(got[fin].view(np.int32).astype(np.int64) - ref[fin].view(np.int32).astype(np.int64))
    same_sign = np.signbit(got[fin]) == np.signbit(ref[fin])
    assert same_sign.all() and ulp.max() <= 2, ulp.max()


# ---- modulation ------------------------------------------------------------------------------------------------------------
# device error <= FEATURE_RATIO x the reference's own worst error vs the float64 truth, per feature.  Measured on an H100: worst
# ratios 2.04 / 1.41 / 2.01 / 1.04, the first and third on an 8-sample message (four wavelet values, P = 8, scale 1).
FEATURE_RATIO = 2.5


def test_modulation_decisions_and_features(AI, oracle):
    want = cases.recorded("test_modulation_pinned")
    excluded, rel_dev, rel_ref, names = [], [], [], []
    for i, (name, x, scale, order) in enumerate(cases.modulation_cases(oracle)):
        decision, (nz, feat) = want[i]
        mine = AI.detect_modulation(x, scale, order)
        f, _ = AI.modulation_features(x, scale, order)
        assert int(f[0]) == nz, name
        if cases.near_threshold(feat):
            excluded.append(name)
        else:
            assert mine == decision, (name, mine, decision)
        if feat is None:
            assert int(f[2]) == 0 or len(x) - nz > 3, name
            continue
        ref = np.array(feat[:4])
        if not np.isfinite(ref).all():
            assert not np.isfinite(f[3:7]).all(), name
            continue
        _, truth = oracle.modulation_features(x.astype(np.complex128), scale, order)
        truth = np.array(truth[:4])
        rel_dev.append(np.abs(f[3:7] - truth) / np.abs(truth))
        rel_ref.append(np.abs(ref - truth) / np.abs(truth))
        names.append(name)
    rel_dev, rel_ref = np.array(rel_dev), np.array(rel_ref)
    worst_dev, worst_ref = rel_dev.max(axis=0), rel_ref.max(axis=0)
    print("modulation: %d messages, %d near a threshold, %d feature sets vs the float64 truth" % (len(want), len(excluded), len(names)))
    print("  worst relative error per feature: device %s (%s), reference %s, ratio %s"
          % (worst_dev, [names[k] for k in rel_dev.argmax(axis=0)], worst_ref, np.round(worst_dev / worst_ref, 3)))
    assert len(excluded) <= 0.05 * len(want), excluded
    # Per message the two errors are independent float32 roundings, and either can be ~0 by chance, so the bound is the
    # reference's own worst distance over the matrix, per feature.
    assert np.all(rel_dev <= FEATURE_RATIO * worst_ref), [names[k] for k in np.nonzero((rel_dev > FEATURE_RATIO * worst_ref).any(axis=1))[0]]


def test_nan_samples_are_dropped_like_the_reference(AI):
    """data[np.abs(data) > 0]: (NaN, 0) and (0, NaN) are dropped and count with the zeros, (inf, NaN) has |x| = inf and stays"""
    from oracle import oracle
    x = cases.modulated(oracle, "FSK", 50, 80, 920)[:4000]
    x[[11, 1000]] = [complex(np.nan, 0.0), complex(0.0, np.nan)]
    assert AI.detect_modulation(x) == "FSK"
    f, _ = AI.modulation_features(x)
    assert int(f[0]) == 3998
    x[[5, 6, 7]] = complex(np.nan, 0.0)
    assert AI.detect_modulation(x) == "OOK" and int(AI.modulation_features(x)[0][0]) == 3995
    y = cases.modulated(oracle, "FSK", 50, 80, 921)[:4000]
    y.view(np.float32)[34:36] = [np.inf, np.nan]
    assert int(AI.modulation_features(y)[0][0]) == 4000


@pytest.mark.parametrize("scale", [1, 4, 8])
def test_cwt_haar_against_float64(scale):
    from oracle import oracle
    from urh_b200.ainterpretation import Wavelet
    rng = np.random.default_rng(scale)
    for n in (4 * scale + 1, 1023, 1024, 1025, 1 << 16):
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        truth = oracle.cwt_haar(x.astype(np.complex128), scale=scale)
        peak = max(np.max(np.abs(truth)), 1e-300) if len(truth) else 1.0
        got = Wavelet.cwt_haar(x.astype(np.complex128), scale=scale)
        assert got.shape == truth.shape and (len(got) == 0 or np.max(np.abs(got - truth)) <= 1e-12 * peak), n
        got32 = Wavelet.cwt_haar(x, scale=scale)
        P = 1 << int(np.log2(n))
        bound = 8 * np.finfo(np.float32).eps * np.log2(P) * peak
        assert got32.shape == truth.shape
        if len(truth):
            assert np.max(np.abs(got32 - truth)) <= bound, n
            assert np.max(np.abs(oracle.cwt_haar(x, scale=scale) - truth)) <= bound, n   # numpy's complex64 path, same bound


def _fft_argmax(x):
    from urh_b200 import _lib
    from urh_b200.device import to_device
    ctx = _lib.default_context()
    x = np.ascontiguousarray(x, dtype=np.complex64)
    d = to_device(x.view(np.float32), ctx)
    idx, P = C.c_int64(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_fft_argmax(ctx.handle, C.c_void_p(d.ptr), len(x), C.byref(idx), C.byref(P)))
    return idx.value, P.value


def test_fft_argmax():
    rng = np.random.default_rng(17)
    checked = 0
    for n in (1, 2, 3, 255, 256, 257, 4095, 4096, 4097, (1 << 20) + 1):
        P = 1 << int(np.log2(n))
        for kind in ("tone+", "tone-", "noise", "zeros"):
            t = np.arange(n)
            if kind == "zeros":
                x = np.zeros(n, np.complex64)
            elif kind == "noise":
                x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
            else:
                b = int(rng.integers(0, max(1, P // 2)))
                b = b if kind == "tone+" else -b
                x = (np.exp(2j * np.pi * b * t / P) + 0.1 * rng.standard_normal(n)).astype(np.complex64)
            k, gotP = _fft_argmax(x)
            assert gotP == P
            if kind == "zeros":
                assert k == 0
                continue
            mag = np.abs(np.fft.fft(x[:P].astype(np.complex128)))
            top2 = np.sort(mag)[-2:] if P > 1 else np.array([0.0, mag[0]])
            bound = 8 * np.finfo(np.float32).eps * np.log2(max(P, 2)) * np.sqrt(np.sum(np.abs(x[:P].astype(np.complex128)) ** 2))
            if top2[1] - top2[0] > bound:
                assert k == int(np.argmax(mag)), (n, kind)
                checked += 1
    assert checked >= 25


# ---- estimate() end to end ----------------------------------------------------------------------------------------------
def test_estimate_end_to_end(AI):
    from oracle import oracle
    want = cases.recorded("test_estimate_pinned")
    for i, (name, iq) in enumerate(cases.estimate_cases(oracle)):
        got = outcome(lambda: AI.estimate(iq.copy()))
        ref = want[i]
        assert (got is None) == (ref is None), (name, got, ref)
        if ref is None:
            continue
        assert set(got) == set(ref), name
        for key in ("modulation_type", "bit_length", "tolerance", "noise"):
            assert got[key] == ref[key], (name, key, got, ref)
        assert float(got["center"]) == float(ref["center"]), (name, got["center"], ref["center"])
