"""GPU: the FIR filter's device entries against the oracle (pinned to the reference by test_oracle.py) on every case of
tests/fir_edge_cases.py, word for word with NaN folded and -0 apart from +0:
* signal_functions.fir_filter on a host array, on a DeviceArray and on the views d[1:] and d[3:] (a view at an odd sample offset
  misaligns the tile's bulk copy);
* urh_fir_filter_shard with history, split where the shard's first m - 1 outputs read the previous shard (a split at m - 1, the
  smallest a neighbour's halo allows, and one sample after each non-finite sample), on tile edges and at n - 1;
* urh_fir_filter_stream with chunks of one and three tiles and one shorter than the m - 1 history (the plan enlarges it), rings of
  two and three;
* Filter(taps, FilterType.custom).work on a few cases.
The C entries return n outputs for n samples, so the cases without taps or samples go only through the Python entries."""
import ctypes as C
import warnings

import numpy as np
import pytest

from fir_edge_cases import GROUPS, cases, folded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from urh_b200 import _lib

    if not _lib.cuda_available():
        pytest.skip("no CUDA device")
    return _lib.default_context()


@pytest.fixture(scope="module")
def by_group():
    groups = {g: [] for g in GROUPS}
    for c in cases():
        groups[c.group].append(c)
    return groups


_EXPECTED = {}


def expected(case, skip=0):
    """the oracle's words for the case's samples from `skip` on, or "ValueError" """
    from oracle import oracle

    key = (case.name, skip)
    if key not in _EXPECTED:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            try:
                _EXPECTED[key] = folded(oracle.fir_filter(case.x[skip:], case.taps))
            except ValueError:
                _EXPECTED[key] = "ValueError"
    return _EXPECTED[key]


def answer(call):
    try:
        return folded(np.asarray(call()))
    except ValueError:
        return "ValueError"


def agrees(got, want):
    if isinstance(got, str) or isinstance(want, str):
        return isinstance(got, str) and isinstance(want, str) and got == want
    return got.shape == want.shape and np.array_equal(got, want)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _c_entry_cases(cs):
    return [c for c in cs if len(c.x) and len(c.taps)]


def shard_splits(case):
    """first samples g0 of a second shard: the smallest a halo of m - 1 samples allows, one sample after each non-finite sample and
    half the history later, tile edges, n - 1"""
    n, m = len(case.x), len(case.taps)
    g = {m - 1, m, 1023, 1024, 1025, 2048, n - 1}
    bad = np.flatnonzero(~np.isfinite(case.x.view(np.float32).reshape(-1, 2)).all(1))
    for p in bad[:4]:
        g |= {int(p) + 1, int(p) + 1 + (m - 1) // 2}
    return sorted(s for s in g if max(1, m - 1) <= s <= n - 1)


@pytest.mark.parametrize("group", GROUPS)
def test_host_array(ctx, by_group, group):
    from urh_b200.cythonext import signal_functions as sf

    bad = [c.name for c in by_group[group] if not agrees(answer(lambda: sf.fir_filter(c.x, c.taps)), expected(c))]
    assert not bad, bad[:20]


@pytest.mark.parametrize("group", GROUPS)
def test_device_array_and_views(ctx, by_group, group):
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import to_device

    bad = []
    for c in by_group[group]:
        d = to_device(c.x, ctx)
        for skip in (0, 1, 3):
            if skip and len(c.x) <= skip:
                continue
            view = d[skip:] if skip else d
            if not agrees(answer(lambda: sf.fir_filter(view, c.taps).get()), expected(c, skip)):
                bad.append((c.name, skip))
    assert not bad, bad[:20]


@pytest.mark.parametrize("group", GROUPS)
def test_shard_with_history(ctx, by_group, group):
    from urh_b200.device import DeviceArray, to_device

    bad, splits = [], 0
    for c in _c_entry_cases(by_group[group]):
        n, m = len(c.x), len(c.taps)
        want = expected(c)
        d_t = to_device(c.taps, ctx)
        d_x = to_device(c.x, ctx)
        for g0 in shard_splits(c):
            h = m - 1
            out = DeviceArray(ctx, (n - g0,), np.complex64)
            ctx.check(ctx.lib.urh_fir_filter_shard(ctx.handle, C.c_void_p(d_x.ptr + 8 * g0), n - g0, int(h > 0), C.c_void_p(d_t.ptr), m,
                                                   C.c_void_p(out.ptr)))
            if not np.array_equal(folded(out.get()), want[2 * g0:]):
                bad.append((c.name, g0))
            splits += 1
        # the first shard: the zero initial state
        out = DeviceArray(ctx, (n,), np.complex64)
        ctx.check(ctx.lib.urh_fir_filter_shard(ctx.handle, C.c_void_p(d_x.ptr), n, 0, C.c_void_p(d_t.ptr), m, C.c_void_p(out.ptr)))
        if not np.array_equal(folded(out.get()), want):
            bad.append((c.name, 0))
    assert not bad, bad[:20]
    assert splits or group == "empty"


@pytest.mark.parametrize("group", GROUPS)
def test_streamed(ctx, by_group, group):
    bad = []
    for c in _c_entry_cases(by_group[group]):
        m = len(c.taps)
        want = expected(c)
        for cs, ring in ((1024, 2), (3 * 1024, 3), (max(1, (m - 1) // 2), 2), (max(1, (m - 1) // 2), 3)):
            y = np.full(len(c.x), np.nan, dtype=np.complex64)
            ctx.check(ctx.lib.urh_fir_filter_stream(ctx.handle, _ptr(c.x), len(c.x), _ptr(c.taps), m, cs, ring, _ptr(y)))
            if not np.array_equal(folded(y), want):
                bad.append((c.name, cs, ring))
    assert not bad, bad[:20]


FILTER_CASES = ["annexg_inf_sample_example", "annexg_padded_inf_tap3_example", "annexg_overflow_nan_example", "overflow_then_neginf_real",
                "subnormal_near_flt_min", "neg_zero_all_terms", "shape_m33_n2049", "large_m12288_n5000", "empty_taps_n3", "empty_taps_n0"]


def test_filter_work(ctx):
    from urh_b200.signalprocessing.Filter import Filter, FilterType

    named = {c.name: c for c in cases()}
    bad = [name for name in FILTER_CASES
           if not agrees(answer(lambda: Filter(named[name].taps, FilterType.custom).work(named[name].x)), expected(named[name]))]
    assert not bad, bad
