"""GPU: the digitizer (grab_pulse_lens and the fused demodulate-and-digitize entry points) against the oracle at its edges.

A  every case of tests/pulse_edge_cases.py (pinned to the reference by tests/test_oracle.py) through grab_pulse_lens on a host
   array, on a DeviceArray, on the device view one float in (d[1:]: not aligned for the paired loads) and streamed
   (urh_grab_pulse_lens_stream, chunks of 1 and 3 tiles, rings of 2 and 3), row for row against oracle.grab_pulse_lens; then each
   table through ppseq_to_bits (urh_ppseq_to_bits) at the case's own bits per symbol against oracle.ppseq_to_bits.
B  multi-level FSK captures (2 .. 256 symbol frequencies) whose thresholds sit on qad levels, so that samples land on and next to
   them, through demod_digitize (resident, on the device and streamed) and demod_center_digitize's stepwise path; PSK captures
   through demod_digitize with Costas loops of order 2, 4 and 8.  qad is compared word for word with NaN folded
   (dense_edge_cases.folded), rows against the oracle's rows on the oracle's qad."""
import ctypes as C

import numpy as np
import pytest

from pulse_edge_cases import TILE, cases
from test_gpu_bits import assert_same, both
from test_gpu_dense_edges import _same, sf  # noqa: F401  (sf: the module fixture)

pytestmark = pytest.mark.gpu

CASES = cases()
STREAMS = [(TILE, 2), (TILE, 3), (3 * TILE, 2), (3 * TILE, 3)]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _code(mod):
    from urh_b200 import _lib as L

    code = L.demod_mod_code(mod)
    return code if code >= 0 else 99


def s_grab(ctx, x, case, cs, ring):
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    k = C.c_int64(0)
    ctx.check(ctx.lib.urh_grab_pulse_lens_stream(ctx.handle, _ptr(x), 0, len(x), case.center, case.tol, _code(case.mod), case.sps,
                                                 case.bps, case.spacing, cs, ring, C.byref(k)))
    return _fetch_pulses(ctx, k.value)


def s_dd(ctx, iq, noise, mod, center, tol, sps, bps, spacing, cs, ring):
    from urh_b200 import _lib as L
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    k = C.c_int64(0)
    q = np.empty(len(iq), np.float32)
    ctx.check(ctx.lib.urh_demod_digitize_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), len(iq), float(noise), _code(mod), float(center),
                                                tol, sps, bps, float(spacing), cs, ring, _ptr(q), C.byref(k)))
    return q, _fetch_pulses(ctx, k.value)


def _rows_equal(got, want, what):
    if not np.array_equal(got, want):
        k = min(len(got), len(want))
        bad = np.flatnonzero((got[:k] != want[:k]).any(axis=1))
        raise AssertionError((what, "rows", len(got), len(want), bad[:4], got[bad[:2]].tolist() if len(bad) else got[k:k + 2].tolist(),
                              want[bad[:2]].tolist() if len(bad) else want[k:k + 2].tolist()))


# ---- A: the named qad cases ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_pulse_edge_case(sf, oracle, ctx, case):  # noqa: F811
    from urh_b200.device import to_device

    x = case.x
    want = oracle.grab_pulse_lens(x, *case.args())
    _rows_equal(sf.grab_pulse_lens(x, *case.args()), want, "host")
    d = to_device(x, ctx)
    _rows_equal(sf.grab_pulse_lens(d, *case.args()), want, "device")
    if len(x) > 1:
        assert d[1:].ptr % 8 != 0
        _rows_equal(sf.grab_pulse_lens(d[1:], *case.args()), oracle.grab_pulse_lens(x[1:], *case.args()), "device view d[1:]")
    for cs, ring in STREAMS:
        _rows_equal(s_grab(ctx, x, case, cs, ring), want, ("stream", cs, ring))
    if case.bps >= 1 and case.sps >= 1 and len(want) <= 8192:
        for pt, wp in ((8, True), (0, False)):
            assert_same(*both(want, case.sps, case.bps, pt, write_pos=wp))


# ---- B: IQ captures with qad on and next to the thresholds --------------------------------------------------------------------------
B_N = 3 * TILE + 777


def _fsk_levels(bps, seed, n=B_N):
    """2^bps symbol frequencies (phase steps (k - (order - 1) / 2) * step), runs of 20 .. 80 samples, silent gaps, unit amplitude;
    every third run at one of the two levels above zero (the thresholds _on_levels picks)"""
    order = 1 << bps
    step = 2.4 / order
    rng = np.random.default_rng(seed)
    runs = rng.integers(20, 80, n // 20 + 1)
    lv = rng.integers(0, order, len(runs))
    lv[::3] = order // 2 + np.arange(len(lv[::3])) % 2 * (order > 2)
    sym = np.repeat(lv, runs)[:n]
    gap = np.repeat(rng.random(len(runs)) < 0.08, runs)[:n]
    ph = 0.3 + np.cumsum((sym - (order - 1) / 2) * step)
    z = np.where(gap, 0.0, np.exp(1j * ph))
    return np.stack([z.real, z.imag], axis=1).astype(np.float32), step


def _on_levels(q, step, order):
    """a center and spacing whose thresholds are qad values the capture holds: center = the most common qad word of the level just
    above zero, spacing = the distance to the most common word of the next level"""
    kept = q[(q != -4.0) & np.isfinite(q)]

    def mode_near(v):
        near = kept[np.abs(kept - v) < step / 4]
        vals, cnt = np.unique(near, return_counts=True)
        return vals[np.argmax(cnt)]

    if order == 2:
        return float(mode_near(step / 2)), 0.1
    c = mode_near(step / 2)
    return float(c), float(np.float32(mode_near(1.5 * step) - c))


@pytest.mark.parametrize("bps", [1, 2, 3, 4, 5, 6, 7, 8])
def test_fsk_levels_on_thresholds(sf, oracle, ctx, bps):  # noqa: F811
    from urh_b200.device import to_device

    order = 1 << bps
    iq, step = _fsk_levels(bps, seed=40 + bps)
    q_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    center, spacing = _on_levels(q_ref, step, order)
    thr = oracle.get_center_thresholds(center, spacing, order)
    assert np.isin(thr, q_ref).any(), "a threshold on a qad level"
    d = to_device(iq, ctx)
    for tol in (0, 3, 33):
        rows_ref = oracle.grab_pulse_lens(q_ref, center, tol, "FSK", 50, bps, spacing)
        for src, what in ((iq, "host"), (d, "device")):
            q, rows = sf.demod_digitize(src, 0.05, "FSK", center, tol, 50, bps, spacing)
            _same(q, q_ref, (bps, tol, what))
            _rows_equal(rows, rows_ref, (bps, tol, what))
        rows_v = sf.demod_digitize(d[1:], 0.05, "FSK", center, tol, 50, bps, spacing)[1]
        _rows_equal(rows_v, oracle.grab_pulse_lens(oracle.afp_demod(iq[1:], 0.05, "FSK", 2), center, tol, "FSK", 50, bps, spacing),
                    (bps, tol, "view"))
        for cs, ring in STREAMS:
            q, rows = s_dd(ctx, iq, 0.05, "FSK", center, tol, 50, bps, spacing, cs, ring)
            _same(q, q_ref, (bps, tol, cs, ring, "stream"))
            _rows_equal(rows, rows_ref, (bps, tol, cs, ring, "stream"))
        assert_same(*both(rows_ref, 50, bps, 8))
    # the detect-center step's stepwise path (bps > 1 always takes it): the center within the one-call tolerance, rows at that center
    c_ref = oracle.detect_center(q_ref)
    for src in (iq, d):
        c, rows, qad = sf.demod_center_digitize(src, 0.05, "FSK", 3, 50, bps, spacing, return_qad=True, stepwise=True)
        _same(qad, q_ref, (bps, "demod_center_digitize"))
        assert (c is None) == (c_ref is None)
        if c is not None:
            assert abs(c - c_ref) <= 2e-6 * max(1.0, abs(c_ref)), (c, c_ref)
            _rows_equal(rows, oracle.grab_pulse_lens(q_ref, c, 3, "FSK", 50, bps, spacing), (bps, "demod_center_digitize"))


@pytest.mark.parametrize("bps", [1, 2, 3])
def test_psk_levels_on_thresholds(sf, oracle, ctx, bps):  # noqa: F811
    from urh_b200.device import to_device

    order = 1 << bps
    rng = np.random.default_rng(60 + bps)
    n = B_N
    runs = rng.integers(40, 120, n // 40 + 1)
    sym = np.repeat(rng.integers(0, order, len(runs)), runs)[:n]
    gap = np.repeat(rng.random(len(runs)) < 0.08, runs)[:n]
    z = np.where(gap, 0.0, np.exp(1j * (0.02 * np.arange(n) + 2 * np.pi * sym / order)))
    iq = np.stack([z.real, z.imag], axis=1).astype(np.float32)
    q_ref = oracle.afp_demod(iq, 0.05, "PSK", order)
    kept = q_ref[(q_ref != -4.0) & np.isfinite(q_ref)]
    vals, cnt = np.unique(kept, return_counts=True)
    top = np.sort(vals[np.argsort(cnt)[-2:]])                # two common qad words: one is the center, the next a threshold
    center, spacing = float(top[0]), float(np.float32(top[1] - top[0]) if order > 2 else 0.1)
    d = to_device(iq, ctx)
    for tol in (0, 5):
        rows_ref = oracle.grab_pulse_lens(q_ref, center, tol, "PSK", 60, bps, spacing)
        for src, what in ((iq, "host"), (d, "device")):
            q, rows = sf.demod_digitize(src, 0.05, "PSK", center, tol, 60, bps, spacing)
            _same(q, q_ref, (bps, tol, what))
            _rows_equal(rows, rows_ref, (bps, tol, what))
        assert_same(*both(rows_ref, 60, bps, 8))

