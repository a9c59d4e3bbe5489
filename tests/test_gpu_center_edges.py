"""GPU: detect_center and its histogram kernels (center.cu) at their edges, against the oracle and numpy.

* the stand-alone detect_center on every array of tests/center_edge_cases.py (host array, device array, device view one sample
  in), with and without max_size: bit-identical to the oracle, None included (its variance is numpy's, replayed by pairwise.cu);
* urh_center_histogram / urh_center_histogram_tiles with caller-chosen (hmin, hstep, nbins) forcing each variant of
  k_hist_interior (one-look-up FAST with |edge| / hstep just below 2^20, the shared-memory loop with the edge table, shared-memory
  counts with the table in global memory, global counts): counts equal np.histogram on the same edges, with every float32 of some
  bins and samples on ru(edge), pred(ru(edge)), f_hi and succ(f_hi); over the same rank windows, among them windows that start or
  end on a tile boundary next to a silent tile and one inside a tile, urh_center_window_stats (k_center_window) equals numpy;
* the fused steps on ASK / FSK captures: demod_detect_center (bitwise off and on), demod_center_digitize one-call and stepwise,
  the certified pick on and off, levels on both sides of the fine histogram's 1.0 clamp, and a strong nearly constant ASK carrier
  whose variance cancels in the double tile sums;
* the device chain's restatement of np.arange (length, edges, the 6000-bin handback) through the state and center it returns."""
import ctypes as C
import math
import os
import zlib

import numpy as np
import pytest

from center_edge_cases import TILE, cases
from conftest import bits_equal, synth_fsk
from test_center_bins_model import Bins, reference_bin

pytestmark = pytest.mark.gpu

CASES = cases()


def _bits(c):
    return None if c is None else int(np.float64(c).view(np.uint64))


def _within(c, ref):
    """the fused steps' documented bound (DESIGN.md §4.4.1)"""
    return abs(c - ref) <= 2e-6 * max(1.0, abs(ref))


@pytest.fixture(scope="module")
def AI():
    from urh_b200.ainterpretation import AutoInterpretation

    return AutoInterpretation


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _ctx():
    from urh_b200 import _lib

    return _lib.default_context()


def _unaligned(x, ctx):
    """a device view of x one float in: not 16-byte aligned, so every kernel takes its scalar loads"""
    from urh_b200.device import to_device

    d = to_device(np.concatenate([np.zeros(1, np.float32), x]), ctx)
    v = d[1:]
    assert v.ptr % 16 != 0
    return d, v


# ---- the stand-alone detect_center ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["host", "device", "unaligned"])
def test_detect_center_edge_cases_bit_identical(AI, oracle, layout):
    from urh_b200.device import to_device

    ctx = _ctx()
    seen = 0
    for name, x, max_size in CASES:
        keep = None
        if layout == "host":
            arr = x
        elif layout == "device":
            arr = to_device(x, ctx)
        else:
            keep, arr = _unaligned(x, ctx)
        for ms in {max_size, None, 777}:
            with np.errstate(all="ignore"):
                want = _bits(oracle.detect_center(x, ms))
            got = _bits(AI.detect_center(arr, ms))
            assert got == want, (name, ms, got, want)
            seen += 1
        del keep
    assert seen >= 2 * len(CASES)


# ---- the histogram entries with caller-chosen edges ------------------------------------------------------------------------------
def _probe_samples(b, rng, exhaustive):
    """float32 samples: every float32 of the given bins, every threshold kind and its neighbours, random samples over a wider range"""
    out = []
    for k in exhaustive:
        f = b.fe[k]
        while f <= b.fe[min(k + 1, b.nbins)] and len(out) < 200_000:
            out.append(f)
            f = np.nextafter(f, np.float32(np.inf))
    ks = np.unique(np.concatenate([np.arange(min(b.nbins + 1, 64)), rng.integers(0, b.nbins + 1, 256), [b.nbins]]))
    for t in list(b.fe[ks]) + [b.f_hi, b.f_min]:
        out += [t, np.nextafter(t, np.float32(-np.inf)), np.nextafter(t, np.float32(np.inf))]
    span = b.edges[-1] - b.edges[0]
    out += list(rng.uniform(b.edges[0] - 0.01 * span, b.edges[-1] + 0.01 * span, 30_000).astype(np.float32))
    s = np.array(out, dtype=np.float32)
    return s[np.isfinite(s)]


def _layout(samples, rng):
    """the samples spread over whole tiles with -4 noise, a silent tile and a partial last tile, shuffled"""
    s = rng.permutation(samples)
    n = max(8 * TILE, int(len(s) * 1.3)) // TILE * TILE + 1234
    x = np.full(n, -4.0, np.float32)
    slots = np.setdiff1d(np.arange(n), np.arange(2 * TILE, 3 * TILE))   # tile 2 stays silent
    x[np.sort(rng.choice(slots, len(s), replace=False))] = s
    return x


HMIN_BETWEEN = 30000.0 + 0.01 * 2.0 ** -9   # float32 spacing at 30000 is 2^-9
HIST_CASES = {
    # name: (hmin, hstep, nbins, bins swept exhaustively); the FAST bound is |edge| / hstep < 2^20
    "fast_just_below_2p20": (1000.0, 1000.0 / (2 ** 20 - 400), 200, (0, 1, 100, 198, 199)),
    "fast_hmin_between_floats_below_2p20": (1000.0 + 0.01 * 2.0 ** -14, 1000.0 / (2 ** 20 - 400), 200, (0, 1, 199)),
    "fast_negative_just_below_2p20": (-1000.5, 1000.5 / (2 ** 20 - 10), 5, (0, 2, 4)),
    "fast_near_zero": (-0.7, 1.4 / 5000, 5000, (0, 2500, 4999)),
    "loop_smem_edges_offset_5000": (4999.0, 1e-3, 3000, (0, 1, 1500, 2999)),
    "loop_smem_edges_past_2p20": (-30000.0, 30000.0 / 2 ** 22, 4000, (0, 3999)),
    # hmin just above a float32, so ru(hmin) lies most of an ulp above it: here the one-look-up guess would be a bin low
    "loop_smem_edges_hmin_between_floats": (HMIN_BETWEEN, HMIN_BETWEEN / 2 ** 23.5, 3000, (0, 1, 1500, 2999)),
    "smem_counts_global_edges": (-3.5, 7.0 / 9000, 9000, (0, 4500, 8999)),
    "smem_counts_12000": (0.25, 1e-4, 12000, (0, 11999)),
    "global_counts": (-2.0, 4.0 / 50_000, 50_000, (0, 25_000, 49_999)),
    "global_counts_offset": (5000.0, 2e-3, 13_000, (0, 12_999)),
    "below_minus4": (-4.75, 0.25, 20, (0, 3, 4, 19)),
}


@pytest.mark.parametrize("name", sorted(HIST_CASES))
def test_histogram_entries_equal_numpy(AI, name):
    from urh_b200.device import to_device

    hmin, hstep, nbins, sweep = HIST_CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    b = Bins(hmin, hstep, nbins)
    samples = _probe_samples(b, rng, sweep)
    if name == "loop_smem_edges_hmin_between_floats":
        # the loop-based variant must take this range: the one-look-up guess misbins some of its samples
        assert b.ratio < 2 ** 24 and any(b.bin_fast(f) != reference_bin(f, b.edges) for f in samples[-30_000:][:3000])
    x = _layout(samples, rng)
    edges = hmin + np.arange(nbins + 1) * hstep
    ctx = _ctx()
    for arr_name, (keep, d) in (("aligned", (None, to_device(x, ctx))), ("unaligned", _unaligned(x, ctx))):
        st = np.zeros(7)
        ctx.check(ctx.lib.urh_center_stats(ctx.handle, C.c_void_p(d.ptr), len(x), -1, st.ctypes.data_as(C.c_void_p)))
        kept = x[x > -4]
        assert int(st[0]) == len(kept)
        windows = [(0, len(kept)), (int(st[1]), int(st[2])), (TILE + 5, TILE + 6), (3 * TILE - 7, min(7 * TILE + 3, len(kept)))]
        # P[t] = kept samples before tile t; tile 2 is silent, so P[2] == P[3] (ranges below -4 keep almost nothing)
        P = np.cumsum(np.concatenate([[0], (x[:8 * TILE] > -4).reshape(8, TILE).sum(axis=1)]))
        assert P[2] == P[3]
        if P[5] - P[4] > 6:
            windows += [(P[3], P[5]),         # r0: the first rank after the silent tile, r1 - 1: the last rank of tile 4
                        (P[1] + 5, P[2]),     # r1 - 1: the last rank before the silent tile
                        (P[1], P[2]),         # exactly tile 1
                        (P[4] + 3, P[5] - 3)]   # inside one tile
        else:
            assert edges[-1] <= -4.0, name   # only a range below detect_center's -4 keeps (almost) nothing
        for r0, r1 in ((int(a), int(b)) for a, b in windows):
            rect = kept[r0:r1]
            want, _ = np.histogram(rect, bins=edges)
            for entry in (ctx.lib.urh_center_histogram_tiles, ctx.lib.urh_center_histogram):
                y = np.zeros(nbins, dtype=np.int64)
                ctx.check(entry(ctx.handle, C.c_void_p(d.ptr), len(x), r0, r1, C.c_double(hmin), C.c_double(hstep), nbins,
                                y.ctypes.data_as(C.c_void_p)))
                bad = np.nonzero(y != want)[0]
                assert len(bad) == 0, (name, arr_name, r0, r1, bad[:5], y[bad[:5]], want[bad[:5]])
            w = np.zeros(5)
            ctx.check(ctx.lib.urh_center_window_stats(ctx.handle, C.c_void_p(d.ptr), len(x), r0, r1, w.ctypes.data_as(C.c_void_p)))
            want_w = (len(rect), float(rect.min()), float(rect.max())) if len(rect) else (0, np.inf, -np.inf)
            assert (w[0], w[1], w[2]) == want_w, (name, arr_name, r0, r1, w)
            # double sums of float32 values (their squares are exact) in any order: within gamma_(n-1) * sum |term| of the exact sum
            r64 = rect.astype(np.float64)
            gamma = (len(rect) - 1) * 2.0 ** -53 / (1 - (len(rect) - 1) * 2.0 ** -53)
            for got, terms in ((w[3], r64), (w[4], r64 * r64)):
                assert abs(got - math.fsum(terms)) <= gamma * np.abs(terms).sum(), (name, arr_name, r0, r1, got, math.fsum(terms))
        del keep


# ---- the fused steps --------------------------------------------------------------------------------------------------------------
SQRT2 = np.float64(np.float32(np.sqrt(2.0)))


def _ask_qad(a):
    """float32 ASK demodulation of the sample (a, 0): sqrtf(a * a) / float(sqrt(2)) in double, rounded to float32"""
    a = np.float32(a)
    return np.float32(np.float64(np.sqrt(np.float32(a * a))) / SQRT2)


def _amplitude_for(q):
    """a float32 amplitude whose ASK qad is exactly q"""
    a = np.float32(float(q) * float(SQRT2))
    for step in range(12):
        for c in (a, np.nextafter(a, np.float32(np.inf)), np.nextafter(a, np.float32(-np.inf))):
            if _ask_qad(c) == np.float32(q):
                return c
        a = np.nextafter(a, np.float32(np.inf)) if step % 2 else np.nextafter(a, np.float32(-np.inf))
    raise AssertionError("no amplitude for %r" % q)


def _ask_capture(levels, noise=0.0, seed=0, phase=True):
    """float32 IQ whose ASK magnitudes are `levels` (float32) up to `noise` (relative, magnitude only)"""
    rng = np.random.default_rng(seed)
    amp = np.asarray(levels, np.float64) * float(SQRT2) * (1.0 + noise * rng.standard_normal(len(levels)))
    ph = rng.uniform(0, 2 * np.pi, len(levels)) if phase else np.zeros(len(levels))
    return np.ascontiguousarray(np.stack([amp * np.cos(ph), amp * np.sin(ph)], axis=1).astype(np.float32))


def _runs(n, lo, hi, seed, run=50):
    rng = np.random.default_rng(seed)
    return np.repeat(np.where(rng.integers(0, 2, n // run + 1) > 0, hi, lo), run)[:n]


def _fused_captures():
    """(name, iq, noise, mod, max_size)"""
    out = [("fsk_bursts", synth_fsk(300_001, seed=3, gap_every=40_000), 0.05, "FSK", None),
           ("fsk_max_size", synth_fsk(5 * TILE + 1, seed=4), 0.05, "FSK", 3 * TILE + 5),
           ("fsk_2048k_minus_1", synth_fsk(40 * TILE - 1, seed=5, gap_every=9000), 0.05, "FSK", None)]
    for name, lo, hi in (("ask_below_1", 0.3, 0.9), ("ask_across_1", 0.6, 1.4), ("ask_above_1", 1.3, 2.2),
                         ("ask_on_1", 0.5, 1.0)):
        lv = _runs(200_000, lo, hi, seed=int(hi * 10))
        out.append((name, _ask_capture(lv, 0.01, seed=1), 0.05, "ASK", None))
    # a strong, nearly constant carrier: var / mean^2 ~ 1e-15 .. 1e-10, where Σx² - n·mean² cancels
    out.append(("ask_carrier_3e4_2e-3", _ask_capture(np.full(200_000, 3e4), 2e-3 / 3e4, seed=2), 0.05, "ASK", None))
    out.append(("ask_carrier_3e4_0.5", _ask_capture(np.full(200_000, 3e4), 0.5 / 3e4, seed=3), 0.05, "ASK", None))
    out.append(("ask_carrier_two_levels_3e4", _ask_capture(_runs(200_000, 3e4, 3e4 + 0.05, seed=4), 4e-3 / 3e4, seed=4), 0.05,
                "ASK", None))
    out.append(("ask_constant", _ask_capture(np.full(100_003, np.float32(0.7)), 0.0, seed=5, phase=False), 0.05, "ASK", None))
    return out


FUSED = _fused_captures()


def _one_call(sf, iq, noise, mod, max_size, certify):
    if certify:
        os.environ.pop("URH_B200_CENTER_NO_CERTIFY", None)
    else:
        os.environ["URH_B200_CENTER_NO_CERTIFY"] = "1"
    try:
        c, rows = sf.demod_center_digitize(iq, noise, mod, 5, 100, max_size=max_size)
        return c, np.asarray(rows).copy()
    finally:
        os.environ.pop("URH_B200_CENTER_NO_CERTIFY", None)


@pytest.mark.parametrize("case", [c[0] for c in FUSED])
def test_fused_steps(AI, sf, oracle, case):
    name, iq, noise, mod, max_size = next(c for c in FUSED if c[0] == case)
    qad_ref = oracle.afp_demod(iq, noise, mod, 2)
    with np.errstate(all="ignore"):
        ref = oracle.detect_center(qad_ref, max_size)
    qad, c = AI.demod_detect_center(iq, noise, mod, max_size)
    assert bits_equal(qad.get(), qad_ref) == 0
    assert (c is None) == (ref is None), (name, c, ref)
    if c is not None:
        assert _within(c, ref), (name, c, ref)
    _, exact = AI.demod_detect_center(iq, noise, mod, max_size, bitwise=True)
    assert _bits(exact) == _bits(ref), (name, exact, ref)
    stepwise, rows_s = sf.demod_center_digitize(iq, noise, mod, 5, 100, max_size=max_size, stepwise=True)
    assert _bits(stepwise) == _bits(c)
    c1, rows1 = _one_call(sf, iq, noise, mod, max_size, True)
    c0, rows0 = _one_call(sf, iq, noise, mod, max_size, False)
    assert _bits(c1) == _bits(c0) and np.array_equal(rows1, rows0), name   # the certificate never changes a result
    assert (c1 is None) == (ref is None), (name, c1, ref)
    if c1 is not None:
        assert _within(c1, ref), (name, c1, ref)
    assert _bits(c1) == _bits(stepwise), (name, c1, stepwise)
    assert np.array_equal(rows1, rows_s)


def test_nearly_constant_carrier_follows_numpy(AI, oracle):
    """where Σx² - n·mean² cancels (var / mean^2 below 2^-14) the fused steps replay numpy's variance: bit-identical centers"""
    for name, iq, noise, mod, max_size in FUSED:
        if not name.startswith(("ask_carrier", "ask_constant")):
            continue
        qad = oracle.afp_demod(iq, noise, mod, 2)
        rect = qad[qad > -4]
        rect = rect[int(0.05 * len(rect)):int(0.95 * len(rect))]
        mean = rect.astype(np.float64).mean()
        assert rect.astype(np.float64).var() < mean * mean * AI.FUSED_VAR_MIN_RATIO, name
        with np.errstate(all="ignore"):
            ref = oracle.detect_center(qad, max_size)
        _, c = AI.demod_detect_center(iq, noise, mod, max_size)
        assert _bits(c) == _bits(ref), (name, c, ref)


# ---- the device chain's np.arange ----------------------------------------------------------------------------------------------
def _chain(iq, noise, mod, max_size=None):
    """urh_demod_center_digitize on a device capture -> (state, center)"""
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device

    ctx = _ctx()
    d = to_device(iq, ctx)
    qad = DeviceArray(ctx, (len(iq),), np.float32)
    center, state, k = C.c_double(0.0), C.c_int(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_demod_center_digitize(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(d.dtype), len(iq), float(noise),
                                                _lib.demod_mod_code(mod), 5, 100, -1 if max_size is None else int(max_size),
                                                C.c_void_p(qad.ptr), C.byref(center), C.byref(state), C.byref(k)))
    return state.value, center.value


def _host_plan(AI, iq, noise, mod, max_size=None):
    """what the chain should decide: the double tile-sum window statistics, np.arange's edges, np.histogram, the peak pick"""
    qad, _ = AI.demod_detect_center(iq, noise, mod, max_size)
    ctx = qad.ctx
    kept = C.c_int64(0)
    from urh_b200 import _lib
    from urh_b200.device import to_device

    d = to_device(iq, ctx)
    ctx.check(ctx.lib.urh_afp_demod_tiles(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(d.dtype), len(iq), float(noise),
                                          _lib.demod_mod_code(mod), C.c_void_p(qad.ptr), 0, C.byref(kept)))
    r0, r1 = AI.center_rank_window(kept.value, max_size)
    w = np.zeros(5)
    ctx.check(ctx.lib.urh_center_window_stats(ctx.handle, C.c_void_p(qad.ptr), len(iq), r0, r1, w.ctypes.data_as(C.c_void_p)))
    st = AI.center_stats_from_window(kept.value, r0, r1, w)
    if not AI.fused_variance_stands(st):
        return 2, None, None
    edges = AI.center_bin_edges(st)
    if edges is None:
        return 0, None, None
    if len(edges) - 1 > 6000:
        return 2, None, len(edges) - 1
    host = qad.get()
    rect = host[host > -4][r0:r1]
    y, _ = np.histogram(rect, bins=edges)
    # a tie that decides which peaks are taken goes back to the host (np.argsort's order among equal counts)
    nb = len(y)
    window = max(2, int(0.05 * nb) + 1)
    peaks = [y[i] for i in range(nb) if y[i] > 0 and all(y[i] > (y[j] if 0 <= j < nb else 0) for d in range(1, window)
                                                          for j in (i - d, i + d))]
    peaks.sort(reverse=True)
    if peaks.count(peaks[0]) > 2 or (len(peaks) > 2 and peaks[0] != peaks[1] and peaks.count(peaks[1]) > 1):
        return 2, None, nb
    return 1, AI.pick_center_from_histogram(y, edges), nb


def _two_levels(lo, hi, n=40_000):
    """ASK qad exactly lo / hi, alternating, so the window holds as many of each"""
    a = np.array([_amplitude_for(lo), _amplitude_for(hi)], np.float32)[np.arange(n) % 2]
    iq = np.ascontiguousarray(np.stack([a, np.zeros(n, np.float32)], axis=1))
    return iq


@pytest.mark.parametrize("case", ["ceil_exact_4096", "bins_6000", "bins_6001", "single_peak", "constant", "three_levels_tie",
                                  "three_levels_top_pair", "close_levels_replayed"])
def test_chain_restates_np_arange(AI, oracle, case):
    q0 = np.float32(2.0 ** -5)   # low enough that var / mean^2 stays above 2^-14 for the two-level cases
    if case == "close_levels_replayed":
        iq = _two_levels(np.float32(0.5), np.float32(0.5 + 2.0 ** -10))   # var / mean^2 ~ 2^-20: the host replays numpy's variance
    elif case == "ceil_exact_4096":
        iq = _two_levels(q0, q0 + np.float32(2.0 ** -10))   # var = 2^-22 exactly: (max + var - min) / var = 4097
    elif case == "bins_6000":
        iq = _two_levels(q0, q0 + np.float32(11185 * 2.0 ** -24))
    elif case == "bins_6001":
        iq = _two_levels(q0, q0 + np.float32(11184 * 2.0 ** -24))
    elif case == "single_peak":
        lv = np.full(30_000, q0, np.float32)
        lv[::7] = np.float32(0.625)
        iq = _ask_capture(lv, 0.0, seed=9, phase=False)
    elif case == "constant":
        iq = _ask_capture(np.full(30_000, q0), 0.0, seed=9, phase=False)
    elif case == "three_levels_tie":   # the second peak ties: the device hands the pick back (state 2)
        lv = np.array([0.25, 0.5, 0.75, 0.5], np.float32)[np.arange(60_000) % 4]
        iq = _ask_capture(lv, 0.0, seed=9, phase=False)
    else:   # exactly two peaks share the top count: both are taken
        lv = np.array([0.25, 0.5, 0.75, 0.5, 0.75], np.float32)[np.arange(60_000) % 5]
        iq = _ask_capture(lv, 0.0, seed=9, phase=False)
    qad_ref = oracle.afp_demod(iq, 0.0, "ASK", 2)
    with np.errstate(all="ignore"):
        ref = oracle.detect_center(qad_ref)
    want_state, want_center, nbins = _host_plan(AI, iq, 0.0, "ASK")
    state, center = _chain(iq, 0.0, "ASK")
    assert state == want_state, (case, state, want_state, nbins)
    if case == "bins_6000":
        assert nbins == 6000
    if case == "bins_6001":
        assert nbins == 6001
    if state == 1:
        assert _bits(center) == _bits(want_center), (case, center, want_center)
        assert _within(center, ref)
    if want_state == 0:
        assert ref is None
    if case.startswith("three_levels"):
        assert state == (2 if case.endswith("tie") else 1)
