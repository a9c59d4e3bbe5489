"""CPU: the oracle's auto-interpretation functions pinned to the reference's own answers on the case matrix of
tests/autointerp_cases.py: get_magnitudes, detect_noise_level, segmentation, plateau lengths, median_filter, detect_center,
detect_modulation with its four variances, and the estimate() dict.  The answers are recorded in tests/golden/ref_autointerp.json
(oracle/cassette.py), so these tests and tests/test_gpu_autointerp.py need nothing outside the repository.  Regenerate after
changing the matrix:

    python -c "import __graft_entry__ as g; g.build()"
    URH_RECORD_GOLDEN=1 python -m pytest tests/test_autointerp_reference_cpu.py
"""
import numpy as np
import pytest

import autointerp_cases as cases
from oracle.cassette import RECORD, Cassette, digest, fingerprint, same


@pytest.fixture
def cassette(request):
    c = Cassette("autointerp", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ref():
    if not RECORD:
        return None
    from oracle import ref_loader
    ns = ref_loader.load_python_layer()
    ns.sf, ns.ut, ns.ai = ref_loader.load_kernels()
    return ns


def outcome(thunk):
    """thunk()'s value, or ("raises", exception class name): the reference raises on some inputs (inf in a quiet chunk)"""
    try:
        return thunk()
    except Exception as e:   # noqa: BLE001 -- the exception is the answer
        return ("raises", type(e).__name__)


def nan_equal(a, b):
    return a == b or (isinstance(a, float) and isinstance(b, float) and np.isnan(a) and np.isnan(b))


def test_magnitudes_pinned(oracle, cassette, ref):
    k = 0
    for iq in cases.magnitude_cases():
        want = cassette.want(lambda: digest(cases.canon(ref.ut.get_magnitudes(iq))))
        assert digest(cases.canon(oracle.get_magnitudes(iq))) == want, (iq.dtype, len(iq))
        k += 1
    assert k == 40


def test_noise_level_pinned(oracle, cassette, ref):
    k = 0
    for name, mags in cases.noise_cases():
        want = cassette.want(lambda: outcome(lambda: ref.AutoInterpretation.detect_noise_level(mags)))
        assert outcome(lambda: oracle.detect_noise_level(mags)) == want, name
        k += 1
    assert k == 240


def test_noise_level_edge_f32_recorded(cassette, ref):
    """the float32 case on the quiet edge: the reference keeps the second chunk loud"""
    want = cassette.want(lambda: ref.AutoInterpretation.detect_noise_level(cases.edge_f32_noise()))
    assert want == 0.01


def test_noise_level_iq_pinned(oracle, cassette, ref):
    for name, iq in cases.noise_iq_cases():
        want = cassette.want(lambda: outcome(lambda: ref.AutoInterpretation.detect_noise_level(ref.ut.get_magnitudes(iq))))
        assert outcome(lambda: oracle.detect_noise_level(oracle.get_magnitudes(iq))) == want, name


def test_segments_pinned(oracle, cassette, ref):
    for name, mags, thr in cases.segment_cases():
        want = cassette.want(lambda: fingerprint(ref.AutoInterpretation.segment_messages_from_magnitudes(mags, thr)))
        assert fingerprint(oracle.segment_messages_from_magnitudes(mags, thr)) == want, name


def test_plateau_lengths_pinned(oracle, cassette, ref):
    for name, rect, center, pct in cases.plateau_cases():
        want = cassette.want(lambda: np.asarray(ref.ai.get_plateau_lengths(rect, center, pct), dtype=np.uint64))
        assert same(oracle.get_plateau_lengths(rect, center, pct), want), name


def test_median_filter_pinned(oracle, cassette, ref):
    for name, data, k in cases.median_cases():
        want = cassette.want(lambda: np.asarray(ref.ai.median_filter(data, k), dtype=np.float32))
        assert same(oracle.median_filter(data, k), want), name


def test_detect_center_pinned(oracle, cassette, ref):
    for name, rect, max_size in cases.center_cases():
        want = cassette.want(lambda: ref.AutoInterpretation.detect_center(rect, max_size=max_size))
        got = oracle.detect_center(rect, max_size=max_size)
        assert (got is None) == (want is None), name
        if got is not None:
            assert float(got) == float(want), name


def test_modulation_pinned(oracle, cassette, ref):
    """decision and features of every message; the oracle's four variances and FSK test equal the reference's to the bit"""
    near = total = 0
    for name, x, scale, order in cases.modulation_cases(oracle):
        want = cassette.want(lambda: (ref.AutoInterpretation.detect_modulation(x.copy(), scale, order),
                                      cases.features_with(ref.Wavelet.cwt_haar, ref.ai.median_filter, x.copy(), scale, order)))
        decision, (nz, feat) = want
        assert oracle.detect_modulation(x, scale, order) == decision, name
        onz, ofeat = oracle.modulation_features(x, scale, order)
        assert onz == nz and (ofeat is None) == (feat is None), name
        if feat is not None:
            assert all(nan_equal(a, b) for a, b in zip(ofeat, feat[:5])), (name, ofeat, feat)
            near += cases.near_threshold(feat)
        total += 1
    assert total == 103
    assert near <= 0.05 * total, near


def test_estimate_pinned(cassette, ref):
    """the reference's estimate() dicts: recorded for tests/test_gpu_autointerp.py (the oracle has no estimate())"""
    k = 0
    from oracle import oracle as o
    for name, iq in cases.estimate_cases(o):
        want = cassette.want(lambda: outcome(lambda: ref.AutoInterpretation.estimate(ref.IQArray(iq.copy()))))
        assert want is None or isinstance(want, dict), (name, want)
        k += 1
    assert k == 40
