"""GPU: speculative digitizing in the detect-center step (UrhSpec, DESIGN.md §4.4.1).

The float32 FSK demodulation pass digitizes its tiles at a guessed threshold t_g; the qad digitizer keeps a tile's result only when
its margin min fl(|s - t_g|) exceeds fl(|c - t_g|) at the detected center c, and digitizes every other tile from qad.  No result
may change: every case runs the step with and without $URH_B200_NO_SPECULATE=1 and compares center, state, qad and pulse rows bit
for bit, checks the rows against the CPU oracle, and asserts through urh_speculate_stats which tiles took which branch."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

TILE = 2048


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _stats(name):
    from urh_b200 import _lib

    ctx = _lib.default_context()
    st = (C.c_int64 * 3)()
    ctx.check(getattr(ctx.lib, name)(ctx.handle, st))
    return list(st)


def _step(sf, d_iq, tol, env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: v for k, v in env.items() if v is not None})
    for k, v in env.items():
        if v is None:
            os.environ.pop(k, None)
    try:
        c, rows, qad = sf.demod_center_digitize(d_iq, 0.05, "FSK", tol, 100, return_qad=True)
        return c, np.asarray(rows).copy(), qad.get(), _stats("urh_speculate_stats"), _stats("urh_center_certify_stats")
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _same(sf, oracle, iq, tol=5, guess=None, certify=True):
    """the step with and without speculation: identical results, rows equal to the oracle's; returns the speculation counters,
    the center and qad"""
    from urh_b200.device import to_device

    d_iq = to_device(iq)
    cert = {"URH_B200_CENTER_NO_CERTIFY": None if certify else "1"}
    c1, r1, q1, st1, cs1 = _step(sf, d_iq, tol, {"URH_B200_NO_SPECULATE": None, "URH_B200_SPECULATE_GUESS": guess, **cert})
    c0, r0, q0, st0, cs0 = _step(sf, d_iq, tol, {"URH_B200_NO_SPECULATE": "1", "URH_B200_SPECULATE_GUESS": None, **cert})
    assert st0 == [0, 0, 0], st0
    assert cs1 == cs0
    assert bits_equal(q1, q0) == 0
    assert c1 == c0
    assert np.array_equal(r1, r0)
    q_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert bits_equal(q1, q_ref) == 0
    if c1 is not None:
        assert np.array_equal(r1, oracle.grab_pulse_lens(q_ref, c1, tol, "FSK", 100))
    n = len(iq)
    nfull = n // TILE
    assert st1[0] == (nfull - 1 if nfull > 1 else 0), (st1, n)
    assert st1[1] + st1[2] == st1[0] and min(st1) >= 0, st1
    return st1, c1, q1, cs1


def _expected_redone(q, c, tg):
    """tiles 1 .. nfull-1 the digitizer must read again: not silent, and margin <= fl(|c - t_g|) (all in float32)"""
    nfull = len(q) // TILE
    t = q[TILE:nfull * TILE].reshape(nfull - 1, TILE)
    margin = np.abs(t - np.float32(tg)).min(axis=1)
    bound = np.abs(np.float32(c) - np.float32(tg))
    silent = (t == np.float32(-4.0)).all(axis=1)
    return int((~silent & ~(margin > bound)).sum())


def _fsk(n, seed, p_one=0.5, dev=0.05, sigma=0.01, gaps=True):
    """the bench recipe in miniature: 2-FSK at +-dev cycles/sample, sps 100, AWGN, bursts and gaps, silence at the end"""
    rng = np.random.default_rng(seed)
    f = np.repeat(np.where(rng.random(n // 100 + 1) < p_one, dev, -dev), 100)[:n]
    x = np.exp(2j * np.pi * np.cumsum(f)) + sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if gaps:
        g = np.arange(n)
        x[(g % 60_000) > 50_000] *= 0.001
        x[int(0.97 * n):] *= 0.001
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))


def test_bench_recipe(sf, oracle):
    st, _, _, _ = _same(sf, oracle, _fsk(1 << 24, seed=1))
    assert st[1] >= 0.95 * st[0], st


@pytest.mark.parametrize("n,tol", [(3_000_001, 5), (1_000_003, 0), (1 << 20, 3000), (TILE, 5), (TILE - 1, 5), (2 * TILE + 1, 5)])
def test_lengths_and_tolerances(sf, oracle, n, tol):
    _same(sf, oracle, _fsk(n, seed=n + tol), tol)


@pytest.mark.parametrize("p_one", [0.95, 0.05])
def test_unbalanced_symbols(sf, oracle, p_one):
    st, _, _, _ = _same(sf, oracle, _fsk(1 << 22, seed=3, p_one=p_one))
    assert st[1] >= 0.9 * st[0], st


@pytest.mark.parametrize("guess", ["0.3", "-0.31", "10", "nan"])
def test_bad_guess_is_redone(sf, oracle, guess):
    st, c, q, _ = _same(sf, oracle, _fsk(1 << 21, seed=5), guess=guess)
    assert c is not None
    # (a NaN guess: no margin exceeds the NaN bound, every tile that is not silent is redone)
    assert st[2] == _expected_redone(q, c, float(guess)), st
    assert st[2] > 0.5 * st[0], st


def test_samples_on_the_thresholds(sf, oracle):
    """three levels: -d, +d and exactly 0.0 (constant phase gives xi == 0 exactly), so c lies near 0 and the guesses can be put
    exactly on sample values, on c itself, and where fl(|s - t_g|) == fl(|c - t_g|) (t_g = c / 2 with s = 0)"""
    n = 1 << 21
    rng = np.random.default_rng(9)
    sym = rng.choice([-1, 1, 0], size=n // 100 + 1, p=[0.46, 0.46, 0.08])
    f = np.repeat(sym * 0.05, 100)[:n]
    x = np.exp(2j * np.pi * np.cumsum(f))
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))
    _, c, q, _ = _same(sf, oracle, iq)
    assert c is not None
    assert (q == 0.0).sum() > 1000
    cf = float(np.float32(c))
    for tg in (0.0, cf, cf / 2, -cf, float(q[12345]), float(np.nextafter(np.float32(cf), np.float32(1.0)))):
        st, c2, q2, _ = _same(sf, oracle, iq, guess=repr(tg))
        assert c2 == c
        assert st[2] == _expected_redone(q2, c, tg), (tg, st)


def test_histogram_pass(sf, oracle):
    """certification off: the histogram pass over qad decides the center, the speculative tiles are verified against it"""
    st, _, _, cs = _same(sf, oracle, _fsk(1 << 22, seed=7), certify=False)
    assert cs[0] == 0 and cs[1] == 0, cs
    assert st[1] >= 0.95 * st[0], st


def test_equal_plateaus_state(sf, oracle):
    """a capture whose certificate does not decide (three equal plateaus): the same results either way"""
    n = 3 * 65536
    ang = np.repeat(np.array([-1.0, 0.0, 1.0]), 65536)
    x = np.exp(1j * np.cumsum(ang))
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))
    _same(sf, oracle, iq)


def test_other_dtypes_not_speculated(sf):
    from urh_b200.device import to_device

    iq = (_fsk(1 << 20, seed=2) * 16000).astype(np.int16)
    c, rows, _, st, _ = _step(sf, to_device(iq), 5, {"URH_B200_NO_SPECULATE": None, "URH_B200_SPECULATE_GUESS": None})
    assert st == [0, 0, 0]
