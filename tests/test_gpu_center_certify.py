"""GPU: the certified peak pick of the one-call step (k_center_certify, DESIGN.md §4.4.1).

The demodulation pass counts the kept samples into a fine histogram; when its bounds decide the two peaks, the histogram pass
over qad is skipped.  The certificate must never change a result: every case runs the step with it and with
$URH_B200_CENTER_NO_CERTIFY=1 (the histogram pass always runs) and compares center, state, qad and pulse rows bit for bit, and
asserts through urh_center_certify_stats which way the step went."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import CAPTURES, bits_equal, load_golden, synth_fsk

pytestmark = pytest.mark.gpu

NB = 4096


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _stats():
    from urh_b200 import _lib

    ctx = _lib.default_context()
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_center_certify_stats(ctx.handle, st))
    return list(st)


def _step(sf, iq, noise, mod, tol, max_size=None, certify=True, **kw):
    if certify:
        os.environ.pop("URH_B200_CENTER_NO_CERTIFY", None)
    else:
        os.environ["URH_B200_CENTER_NO_CERTIFY"] = "1"
    try:
        c, rows, qad = sf.demod_center_digitize(iq, noise, mod, tol, 100, max_size=max_size, return_qad=True, **kw)
        return c, np.asarray(rows).copy(), np.asarray(qad if isinstance(qad, np.ndarray) else qad.get()), _stats()
    finally:
        os.environ.pop("URH_B200_CENTER_NO_CERTIFY", None)


def _same(sf, iq, noise, mod, tol=5, max_size=None, **kw):
    """the step with and without the certificate: identical results; returns the certificate's counter"""
    c1, r1, q1, st1 = _step(sf, iq, noise, mod, tol, max_size, True, **kw)
    c0, r0, q0, st0 = _step(sf, iq, noise, mod, tol, max_size, False, **kw)
    assert st0[0] == 0 and st0[1] == 0, st0          # the switch turns the fine histogram off
    assert st1[1] == NB, st1                          # collected on every unsharded one-call step
    assert bits_equal(q1, q0) == 0
    assert c1 == c0
    assert np.array_equal(r1, r0)
    if st1[0] == 1:
        assert c1 is not None and st1[2] >= 0
    return st1


def _fsk(n, seed, dev=0.05, sigma=0.01, dtype=np.float32):
    """the bench recipe in miniature: 2-FSK at +-dev cycles/sample, bursts and gaps, silence at the end"""
    rng = np.random.default_rng(seed)
    f = np.repeat(np.where(rng.integers(0, 2, n // 100 + 1) > 0, dev, -dev), 100)[:n]
    x = np.exp(2j * np.pi * np.cumsum(f)) + sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    g = np.arange(n)
    x[(g % 60_000) > 50_000] *= 0.001
    x[int(0.97 * n):] *= 0.001
    iq = np.stack([x.real, x.imag], axis=1)
    if dtype == np.int16:
        iq = iq * 16000
    elif dtype == np.int8:
        iq = iq * 100
    elif dtype == np.uint8:
        iq = iq * 100 + 127
    elif dtype == np.uint16:
        iq = iq * 16000 + 32767
    return np.ascontiguousarray(iq.astype(dtype))


NOISE = {np.float32: 0.05, np.int16: 1000.0, np.uint16: 1000.0, np.int8: 5.0, np.uint8: 5.0}


def test_bench_like_capture_certifies(sf):
    st = _same(sf, _fsk(1 << 22, seed=1), 0.05, "FSK")
    assert st[0] == 1, st


@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.uint16, np.int8, np.uint8])
@pytest.mark.parametrize("mod", ["FSK", "ASK"])
@pytest.mark.parametrize("tol", [0, 5])
@pytest.mark.parametrize("max_size", [None, 300_000])
def test_dtypes_modulations(sf, dtype, mod, tol, max_size):
    n = 1_234_567
    iq = _fsk(n, seed=11, dtype=dtype)
    if mod == "ASK":
        env = np.repeat(np.random.default_rng(3).integers(0, 2, n // 100 + 1), 100)[:n] * 0.6 + 0.3
        mid = {np.uint8: 127, np.uint16: 32767}.get(dtype, 0)
        iq = ((iq.astype(np.float64) - mid) * env[:, None] + mid).astype(dtype)
    st = _same(sf, iq, NOISE[dtype], mod, tol, max_size)
    if mod == "FSK" and dtype == np.float32:
        assert st[0] == 1, st


# n around tile (2048) and slab (64 slabs: 8-tile minimum, then ntiles / 64) boundaries
@pytest.mark.parametrize("n", [2047, 2049, 8 * 2048 + 1, 64 * 8 * 2048 - 1, 64 * 8 * 2048 + 2049, 1_000_003, 3 << 20])
def test_tile_and_slab_boundaries(sf, n):
    _same(sf, _fsk(n, seed=n), 0.05, "FSK")


@pytest.mark.parametrize("chunk", [2048, 100_000, 1 << 24])
def test_streamed_host_path(sf, chunk):
    from urh_b200 import _lib
    from urh_b200.device import PinnedArray

    iq = _fsk(1_500_001, seed=7)
    pinned = PinnedArray(iq.shape, iq.dtype, _lib.default_context())
    pinned.array[...] = iq
    try:
        st = _same(sf, pinned.array, 0.05, "FSK", chunk_samples=chunk)
        assert st[0] == 1, st
    finally:
        pinned.free()


def test_ask_with_infinite_samples(sf):
    iq = _fsk(300_000, seed=5)
    env = np.repeat(np.random.default_rng(1).integers(0, 2, 3001), 100)[:300_000] * 0.6 + 0.3
    iq = (iq * env[:, None]).astype(np.float32)
    iq[1000:1010, 0] = np.inf
    iq[5000, 1] = -np.inf
    _same(sf, iq, 0.05, "ASK")


@pytest.mark.parametrize("name", CAPTURES)
def test_golden_captures(sf, name):
    g = load_golden("capture_" + name)
    mod = g["meta"]["mod"]
    if mod not in ("ASK", "FSK"):
        pytest.skip("ASK/FSK only")
    _same(sf, g["iq"], float(g["noise"]), mod)


def test_equal_plateaus(sf):
    """three plateaus of equal population before the rank trim: whichever way the certificate goes, the result equals the
    histogram pass and the stepwise path"""
    n = 3 * 65536
    ang = np.repeat(np.array([-1.0, 0.0, 1.0]), 65536)
    x = np.exp(1j * np.cumsum(ang))
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))
    _same(sf, iq, 0.05, "FSK")
    c1, r1 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100)
    c2, r2 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100, stepwise=True)
    assert c1 == c2 and np.array_equal(r1, r2)


def test_certified_equals_stepwise(sf):
    iq = synth_fsk(1_234_567, seed=11, gap_every=90_000)
    c1, r1 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100)
    c2, r2 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100, stepwise=True)
    assert abs(c1 - c2) <= 1e-9 * max(1.0, abs(c2))
    if c1 == c2:
        assert np.array_equal(r1, r2)
