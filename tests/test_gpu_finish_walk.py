"""GPU: the pulse-table finish (finish.cu) where its warp walks are stressed: more rows than the first guess of the row buffer, more
than 32 firings in one tile, and a redo pass after speculation that digitizes every tile with several tiles per warp."""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _flicker(n, seed, max_run=4):
    """qad whose class changes every 1..max_run samples, with some noise samples (FSK sentinel -4)"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_run + 1, n)
    vals = rng.choice(np.array([-0.5, 0.5, -4.0], np.float32), len(lens), p=[0.45, 0.45, 0.1])
    return np.repeat(vals, lens)[:n].astype(np.float32)


def _fast_fsk(n, seed, sps):
    """2-FSK at +-0.05 cycles/sample with sps samples per symbol: tens to hundreds of firings per 2048-sample tile"""
    rng = np.random.default_rng(seed)
    f = np.repeat(np.where(rng.integers(0, 2, n // sps + 1) > 0, 0.05, -0.05), sps)[:n]
    x = np.exp(2j * np.pi * np.cumsum(f)) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    x[(np.arange(n) % 100_000) > 90_000] *= 0.001
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))


def test_row_buffer_regrowth(sf, oracle):
    """a fresh context sizes the row buffer to n/64 + 1024 rows; tolerance 0 on a flickering signal needs far more, so the finish
    regrows the buffer and repeats its row stage"""
    from urh_b200 import _lib
    from urh_b200.device import to_device

    n = 1 << 20
    x = _flicker(n, seed=7)
    ctx = _lib.Context(0)
    try:
        d = to_device(x, ctx)
        for mod in ("FSK", "ASK"):
            rows = sf.grab_pulse_lens(d, 0.0, 0, mod, 100)
            ref = oracle.grab_pulse_lens(x, 0.0, 0, mod, 100)
            assert len(ref) > n // 64 + 1024
            assert np.array_equal(rows, ref), mod
        del d
    finally:
        ctx.close()


@pytest.mark.parametrize("tol", [0, 1, 5, 31, 32, 33])
def test_many_firings_per_tile_grab(sf, oracle, tol):
    x = _flicker(300_001, seed=tol, max_run=6)
    for mod in ("FSK", "ASK"):
        assert np.array_equal(sf.grab_pulse_lens(x, 0.0, tol, mod, 8), oracle.grab_pulse_lens(x, 0.0, tol, mod, 8)), mod


@pytest.mark.parametrize("tol,sps", [(0, 3), (1, 4), (2, 10)])
def test_many_firings_per_tile_demod_digitize(sf, oracle, tol, sps):
    iq = _fast_fsk(500_003, seed=sps, sps=sps)
    qad, rows = sf.demod_digitize(iq, 0.05, "FSK", 0.0, tol, sps)
    q_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert bits_equal(qad, q_ref) == 0
    ref = oracle.grab_pulse_lens(q_ref, 0.0, tol, "FSK", sps)
    assert len(ref) > 32 * (len(iq) // 2048)
    assert np.array_equal(rows, ref)


@pytest.mark.parametrize("tol,sps", [(0, 3), (1, 4), (2, 10)])
def test_many_firings_per_tile_one_call(sf, oracle, tol, sps):
    iq = _fast_fsk(500_003, seed=sps, sps=sps)
    center, rows, qad = sf.demod_center_digitize(iq, 0.05, "FSK", tol, sps, return_qad=True)
    q_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert bits_equal(qad, q_ref) == 0
    c_ref = oracle.detect_center(q_ref)
    assert center is not None and c_ref is not None
    assert abs(center - c_ref) <= 2e-6 * max(1.0, abs(c_ref))
    ref = oracle.grab_pulse_lens(q_ref, center, tol, "FSK", sps)
    assert len(ref) > 32 * (len(iq) // 2048)
    assert np.array_equal(rows, ref)


def test_every_tile_redone(sf, oracle):
    """a NaN guess proves no tile: the redo pass after speculation digitizes every tile that is not silent, and at 2^26 samples its
    grid (one resident wave of warps) runs several tiles per warp"""
    import test_gpu_speculate as spec

    n = 1 << 26
    iq = spec._fsk(n, seed=9)
    st, c, q, _ = spec._same(sf, oracle, iq, guess="nan")
    assert c is not None
    assert st[2] == spec._expected_redone(q, c, float("nan")), st
    assert st[2] > 0.75 * st[0], st   # all but the silent tiles (gaps and the silent tail)
