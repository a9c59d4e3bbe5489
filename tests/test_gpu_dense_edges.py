"""GPU: the ASK/FSK dense pass (k_dense_iq, k_fsk_fifo) against the oracle at the inputs where it can go wrong.

qad is compared word for word with NaN folded to one word (dense_edge_cases.folded: the payload is not pinned), pulse rows with
oracle.grab_pulse_lens of the oracle's qad.  Which kernel a sample reaches: tile 0 and the last partial tile run k_dense_iq; full
tiles 1 .. nfull - 1 of an aligned FSK capture with a binary digitizer run k_fsk_fifo; a device view one sample in (d[1:]) is not
aligned for the vector loads and runs k_dense_iq only.  (A host array is copied to a fresh, aligned device buffer, so a host view
iq[1:] still takes the fast kernel.)

A  non-finite, huge and subnormal float32 samples at tile edges, inside tile 0 and the last tile, at even and odd positions, through
   afp_demod, demod_digitize, demod_center_digitize and the streamed entry points (the sample on a chunk's last position, so the
   next chunk's halo carries it).  An infinite part takes the reference's Annex G recovery of the float complex product.
B  magnitudes exactly on the noise gate mag <= noise^2, in every dtype, with the noise just above and below; float32 samples where
   a contracted magnitude (fma) would land on the other side of the gate.
C  the fast kernel's operands at the edges of its packed-division window [2^-61, 2^61), at |im/re| = 0.4375, with zero parts and
   with subnormal products.
D  the fused digitizer: every dtype, ASK and FSK, 1..3 bits per symbol, tolerances 0..64, with and without qad, aligned and offset.
E  a 2 M-sample float32 2-FSK capture with a hundred (x, +-inf) samples, through the one-call detect-center step."""
import ctypes as C

import numpy as np
import pytest

from conftest import synth_fsk
from dense_edge_cases import FMAX, INF, NAN, SUB, TINY, folded, fsk_tone

pytestmark = pytest.mark.gpu

TILE = 2048
DTYPES = [np.float32, np.int16, np.uint16, np.int8, np.uint8]


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _dev(iq, ctx):
    from urh_b200.device import to_device

    return to_device(np.ascontiguousarray(iq), ctx)


def _host(a):
    return a if a is None or isinstance(a, np.ndarray) else a.get()


def _same(got, want, what):
    g, w = folded(_host(got)), folded(want)
    bad = np.flatnonzero(g != w)
    assert len(bad) == 0, (what, len(bad), bad[:8], [hex(x) for x in g[bad[:4]]], [hex(x) for x in w[bad[:4]]])


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _code(mod):
    from urh_b200 import _lib as L

    return L.MOD_ASK if mod == "ASK" else L.MOD_FSK


def s_afp(ctx, iq, noise, mod, cs, ring):
    from urh_b200 import _lib as L

    out = np.empty(len(iq), np.float32)
    ctx.check(ctx.lib.urh_afp_demod_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), len(iq), float(noise), _code(mod), cs, ring, _ptr(out)))
    return out


def s_dd(ctx, iq, noise, mod, center, tol, sps, cs, ring):
    from urh_b200 import _lib as L
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    k = C.c_int64(0)
    q = np.empty(len(iq), np.float32)
    ctx.check(ctx.lib.urh_demod_digitize_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), len(iq), float(noise), _code(mod), float(center),
                                                tol, sps, 1, 0.1, cs, ring, _ptr(q), C.byref(k)))
    return q, _fetch_pulses(ctx, k.value)


def _check_demod(sf, oracle, ctx, iq, noise, mod, center=None, tol=3, sps=50, views=True):
    """afp_demod and demod_digitize (qad and rows, with and without qad) of host iq, of the same capture on the device, and of the
    device view one sample in, against the oracle"""
    if center is None:
        center = 0.0 if mod == "FSK" else 0.5
    d = _dev(iq, ctx)
    assert d.ptr % 16 == 0
    layouts = [(iq, iq), (d, iq)]
    if views:
        assert d[1:].ptr % 16 != 0
        layouts.append((d[1:], iq[1:]))
    for arr, ref in layouts:
        q_ref = oracle.afp_demod(ref, noise, mod, 2)
        rows_ref = oracle.grab_pulse_lens(q_ref, center, tol, mod, sps)
        what = (mod, noise, type(arr).__name__, len(arr))
        _same(sf.afp_demod(arr, noise, mod, 2), q_ref, what + ("afp_demod",))
        q, rows = sf.demod_digitize(arr, noise, mod, center, tol, sps)
        _same(q, q_ref, what + ("demod_digitize",))
        assert np.array_equal(rows, rows_ref), what + ("rows",)
        _, rows = sf.demod_digitize(arr, noise, mod, center, tol, sps, return_qad=False)
        assert np.array_equal(rows, rows_ref), what + ("rows without qad",)


def _check_center(sf, oracle, ctx, iq, noise, mod, tol=5, sps=50):
    """demod_center_digitize (one call) from the host and from the device: qad words, the center within the one-call tolerance and
    the rows at that center"""
    q_ref = oracle.afp_demod(iq, noise, mod, 2)
    c_ref = oracle.detect_center(q_ref)
    for src in (iq, _dev(iq, ctx)):
        center, rows, qad = sf.demod_center_digitize(src, noise, mod, tol, sps, return_qad=True)
        _same(qad, q_ref, (mod, type(src).__name__, "demod_center_digitize"))
        assert (center is None) == (c_ref is None), (center, c_ref)
        if center is None:
            assert len(rows) == 0
            continue
        assert abs(center - c_ref) <= 2e-6 * max(1.0, abs(c_ref)), (center, c_ref)
        assert np.array_equal(rows, oracle.grab_pulse_lens(q_ref, center, tol, mod, sps)), (mod, type(src).__name__)


# ---- A: non-finite samples -------------------------------------------------------------------------------------------------------
A_N = 5 * TILE + 777
A_VALUES = [(0.5, INF), (-0.5, -INF), (INF, INF), (0.0, -INF), (-INF, 0.5), (INF, -0.0), (NAN, 0.5), (0.5, NAN), (1e30, -1e30),
            (FMAX, -FMAX), (SUB, 1.0), (-TINY, -0.0)]
# even: a lane's first sample (2048k: lane 0, whose predecessor comes from the previous tile); odd: a lane's second sample
# (2048k - 1: the predecessor lane 0 of the next tile takes; 4095 and 8191 end a chunk of 4096 samples)
A_POSITIONS = {"even": [100, TILE, 2 * TILE, 2 * TILE + 500, 4 * TILE, 5 * TILE, A_N - 300],
               "odd": [101, TILE - 1, 2 * TILE - 1, 2 * TILE + 777, 3 * TILE - 1, 4 * TILE - 1, 5 * TILE - 1, A_N - 1]}


def _a_capture(value, where):
    iq = fsk_tone(A_N, seed=21)
    env = np.repeat(np.random.default_rng(22).choice([0.4, 1.0], A_N // 40 + 1), 40)[:A_N]
    iq *= env[:, None].astype(np.float32)
    iq[A_POSITIONS[where]] = value
    return iq


@pytest.mark.parametrize("where", ["even", "odd"])
@pytest.mark.parametrize("value", A_VALUES, ids=repr)
def test_nonfinite_samples(sf, oracle, ctx, value, where):
    iq = _a_capture(value, where)
    for mod in ("ASK", "FSK"):
        _check_demod(sf, oracle, ctx, iq, 0.05, mod)
        q_ref = oracle.afp_demod(iq, 0.05, mod, 2)
        rows_ref = oracle.grab_pulse_lens(q_ref, 0.0 if mod == "FSK" else 0.5, 3, mod, 50)
        for ring in (2, 3):
            _same(s_afp(ctx, iq, 0.05, mod, 2 * TILE, ring), q_ref, (mod, ring, "afp stream"))
            q, rows = s_dd(ctx, iq, 0.05, mod, 0.0 if mod == "FSK" else 0.5, 3, 50, 2 * TILE, ring)
            _same(q, q_ref, (mod, ring, "demod_digitize stream"))
            assert np.array_equal(rows, rows_ref), (mod, ring)
        # an infinite ASK magnitude is an infinite qad sample, which detect_center's bin edges do not take: FSK angles stay finite
        if not np.isinf(q_ref).any():
            _check_center(sf, oracle, ctx, iq, 0.05, mod)


def test_reference_table_values(sf, oracle):
    """the reference's angles for an infinite imaginary part (the Annex G recovery) on the generic and the fast kernel"""
    from dense_edge_cases import REFERENCE_TABLE

    for prev, cur, word in REFERENCE_TABLE:
        iq = fsk_tone(4 * TILE, seed=5)
        for at in (50, TILE + 50, 2 * TILE + 51):   # tile 0 (generic), a full middle tile (fast), the other lane slot
            iq[at - 1] = prev
            iq[at] = cur
        q = sf.afp_demod(iq, 0.05, "FSK", 2)
        for at in (50, TILE + 50, 2 * TILE + 51):
            assert q[at].view(np.uint32) == word, (prev, cur, at, hex(q[at].view(np.uint32)))
        _same(q, oracle.afp_demod(iq, 0.05, "FSK", 2), (prev, cur))


# ---- B: the noise gate at equality ------------------------------------------------------------------------------------------------
B_N = 4 * TILE + 100
B_INT = {np.int8: ([(3, 4), (-3, 4), (4, -3), (0, 5), (-5, 0)], 5.0, 100),
         np.uint8: ([(3, 4), (4, 3), (0, 5), (5, 0)], 5.0, 100),
         np.int16: ([(3000, 4000), (-4000, 3000), (0, -5000), (5000, 0)], 5000.0, 20000),
         np.uint16: ([(3000, 4000), (4000, 3000), (0, 5000), (5000, 0)], 5000.0, 20000)}


def _f32_gate_samples(k=6, seed=2):
    """float32 (re, im, noise) with RN(RN(re^2) + RN(im^2)) or RN(fma(re, re, RN(im^2))) == RN(noise^2) and the other one on the
    other side of the gate: a contracted magnitude flips the gate for these samples"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < k:
        re = rng.uniform(0.3, 1.0, 4096).astype(np.float32)
        im = rng.uniform(0.3, 1.0, 4096).astype(np.float32)
        m = re * re + im * im                       # float32: each step rounded
        a, b = re.astype(np.float64) ** 2, (im * im).astype(np.float64)
        s = a + b
        bb = s - a
        exact = ((a - (s - bb)) + (b - bb)) == 0    # the float64 sum is exact, so its float32 rounding is the fma's
        f = s.astype(np.float32)
        for i in np.flatnonzero(exact & (f != m)):
            target = m[i] if f[i] > m[i] else f[i]  # gated as the reference computes it, not contracted, or the other way round
            nz = np.float32(np.sqrt(np.float64(target)))
            for cand in (nz, np.nextafter(nz, np.float32(0)), np.nextafter(nz, np.float32(2))):
                if np.float32(cand * cand) == target:
                    out.append((float(re[i]), float(im[i]), float(cand)))
                    break
            if len(out) == k:
                break
    return out


def test_f32_gate_samples_flip_under_contraction():
    for re, im, nz in _f32_gate_samples():
        re, im, nz = np.float32(re), np.float32(im), np.float32(nz)
        nsq = nz * nz
        plain = (re * re + im * im) <= nsq
        fused = np.float32(np.float64(re) ** 2 + np.float64(im * im)) <= nsq
        assert plain != fused


def _b_capture(dtype, samples, scale, seed):
    rng = np.random.default_rng(seed)
    if dtype == np.float32:
        iq = fsk_tone(B_N, seed=seed) * np.float32(4.0)
    else:
        base = synth_fsk(B_N, sps=40, seed=seed).astype(np.float64) * 0.9 * scale
        if dtype in (np.uint8, np.uint16):
            base = np.abs(base) + scale * 0.2
        iq = np.clip(np.round(base), np.iinfo(dtype).min, np.iinfo(dtype).max).astype(dtype)
    at = rng.random(B_N) < 0.15
    at[rng.integers(0, B_N, 40)] = True
    pick = rng.integers(0, len(samples), int(at.sum()))
    iq[at] = np.array(samples, dtype=iq.dtype)[pick]
    return iq


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_noise_gate_at_equality(sf, oracle, ctx, dtype):
    if dtype == np.float32:
        cases = [([(re, im), (-re, im), (re, -im)], nz) for re, im, nz in _f32_gate_samples()]
        scale = 1
    else:
        samples, nz, scale = B_INT[dtype]
        cases = [(samples, nz)]
    for samples, nz in cases:
        iq = _b_capture(dtype, samples, scale, seed=len(samples) + int(nz))
        f = np.float32(nz)
        for noise in (f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(0))):
            for mod in ("ASK", "FSK"):
                center = 0.0 if mod == "FSK" else float(np.median(oracle.afp_demod(iq, 0.0, "ASK", 2)))
                _check_demod(sf, oracle, ctx, iq, float(noise), mod, center=center)


# ---- C: the fast kernel's operand edges ---------------------------------------------------------------------------------------------
def _ulps(x):
    x = np.float32(x)
    return [float(np.nextafter(x, np.float32(0))), float(x), float(np.nextafter(x, np.float32(np.inf)))]


def _c_operands():
    """products (with the predecessor (1, 0) the product is the sample itself): window edges, the |im/re| = 0.4375 branch, zero parts"""
    edges = _ulps(2.0 ** -61) + _ulps(2.0 ** 61)
    ops = []
    for e in edges:
        for other in edges + [e * 0.25, e * 0.5, e * 2.0, 1.0, 0.0, -0.0]:
            ops += [(e, other), (other, e)]
    for re in (1.0, 16.0, 2.0 ** -40, 2.0 ** 40):
        for im in _ulps(re * 0.4375):
            ops += [(re, im), (im, re)]
    for x in (1.0, 0.3, 2.0 ** -61, 2.0 ** 61):
        ops += [(x, 0.0), (x, -0.0), (0.0, x), (-0.0, x)]
    return [(s * a, t * b) for a, b in ops for s in (1.0, -1.0) for t in (1.0, -1.0)
            if (np.float32(a) * np.float32(a) + np.float32(b) * np.float32(b)) > 0]   # noise 0: not gated


def test_fast_operand_edges(sf, oracle, ctx):
    ops = np.array(_c_operands(), dtype=np.float32)
    n = 8 * TILE
    iq = np.zeros((n, 2), np.float32)
    iq[:, 0] = 1.0                                        # (1, 0) at even positions
    rng = np.random.default_rng(8)
    iq[1::2] = ops[rng.integers(0, len(ops), n // 2)]     # an operand at every odd position (its successor sees its conjugate)
    iq[TILE + 1: TILE + 1 + 2 * len(ops): 2] = ops        # every operand at least once in a full middle tile
    # subnormal products: tiny normal samples in a row (their magnitudes stay nonzero at noise 0)
    tiny = np.array([(2.0 ** -70, 2.0 ** -72), (-(2.0 ** -71), 2.0 ** -70), (2.0 ** -74, -(2.0 ** -75)), (2.0 ** -72, 0.0)], np.float32)
    iq[3 * TILE + 100: 3 * TILE + 400] = tiny[rng.integers(0, len(tiny), 300)]
    assert np.all(np.abs(iq[iq != 0]) >= np.float32(2.0 ** -75))
    _check_demod(sf, oracle, ctx, iq, 0.0, "FSK")


@pytest.mark.parametrize("dtype", [np.int16, np.uint16, np.int8, np.uint8], ids=lambda d: np.dtype(d).name)
def test_fast_zero_imaginary_products(sf, oracle, ctx, dtype):
    """integer samples on the axes: products with a zero imaginary part take the packed path (ALLOW_Y0), zero real parts leave it"""
    big = 100 if np.dtype(dtype).itemsize == 1 else 20000
    top = np.iinfo(dtype).max
    vals = [(big, 0), (0, big), (1, 0), (0, 1), (big, big), (top, 0), (7, 0)]
    if np.issubdtype(dtype, np.signedinteger):
        vals += [(-big, 0), (0, -big), (-1, 0), (0, -1), (np.iinfo(dtype).min, 0), (big, -big)]
    vals = np.array(vals, dtype=dtype)
    rng = np.random.default_rng(9)
    iq = vals[rng.integers(0, len(vals), 6 * TILE + 300)]
    _check_demod(sf, oracle, ctx, iq, 0.0, "FSK")


# ---- D: the fused digitizer matrix -------------------------------------------------------------------------------------------------
D_SIZES = [3, 2047, 2049, 3 * TILE, 100_000]
D_NOISE = {np.float32: 0.05, np.int16: 1000.0, np.uint16: 1000.0, np.int8: 5.0, np.uint8: 5.0}


def _levels_capture(n, dtype, mod, order, seed, wide=False):
    """symbols of `order` levels in runs of 1..150 samples, with gaps below the noise gate; wide: complex white noise"""
    rng = np.random.default_rng(seed)
    if wide:
        z = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        z *= 0.3
    else:
        runs = rng.integers(1, 150, n // 2 + 2)
        lvl = np.repeat(rng.integers(0, order, len(runs)), runs)[:n]
        gap = np.repeat(rng.random(len(runs)) < 0.1, runs)[:n]
        if mod == "FSK":
            z = np.exp(1j * np.cumsum((2 * lvl - (order - 1)) * 0.05))
        else:
            z = (0.2 + 0.6 * (lvl + 0.5) / order) * np.exp(0.6j)
        z = np.where(gap, 0.0, z) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    iq = np.stack([z.real, z.imag], axis=1)
    if dtype == np.float32:
        return iq.astype(np.float32)
    scale = 100 if np.dtype(dtype).itemsize == 1 else 20000
    iq = iq * scale
    if np.issubdtype(dtype, np.unsignedinteger):
        iq = iq + (0 if mod == "ASK" and not wide else np.iinfo(dtype).max // 2 + 1)
    return np.clip(np.round(iq), np.iinfo(dtype).min, np.iinfo(dtype).max).astype(dtype)


def _thresholds(q, mod, order):
    """a center and spacing that put the order - 1 thresholds inside the kept samples"""
    kept = q[q != (0.0 if mod == "ASK" else -4.0)]
    kept = kept[np.isfinite(kept)]
    c = np.float32(np.median(kept))
    sp = np.float32((np.percentile(kept, 95) - np.percentile(kept, 5)) / order)
    return float(c), float(max(sp, np.float32(1e-3)))


@pytest.mark.parametrize("mod", ["ASK", "FSK"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_fused_digitizer_matrix(sf, oracle, ctx, dtype, mod):
    noise = D_NOISE[dtype]
    sps = 50
    for bps in (1, 2, 3):
        order = 1 << bps
        for wide in (False, True):
            big = _levels_capture(D_SIZES[-1] + 1, dtype, mod, order, seed=100 * bps + wide, wide=wide)
            nz = 0.0 if wide else noise
            center, spacing = _thresholds(oracle.afp_demod(big, nz, mod, 2), mod, order)
            d = _dev(big, ctx)
            for n in (D_SIZES if not wide else [3 * TILE, D_SIZES[-1]]):
                for arr, ref in ((big[:n], big[:n]), (d[1: n + 1], big[1: n + 1])):
                    q_ref = oracle.afp_demod(ref, nz, mod, 2)
                    for tol in (0, 1, 5, 64):
                        rows_ref = oracle.grab_pulse_lens(q_ref, center, tol, mod, sps, bps, spacing)
                        what = (bps, wide, n, type(arr).__name__, tol)
                        q, rows = sf.demod_digitize(arr, nz, mod, center, tol, sps, bps, spacing)
                        _same(q, q_ref, what)
                        assert np.array_equal(rows, rows_ref), what
                        _, rows = sf.demod_digitize(arr, nz, mod, center, tol, sps, bps, spacing, return_qad=False)
                        assert np.array_equal(rows, rows_ref), what + ("without qad",)


# ---- E: end to end ----------------------------------------------------------------------------------------------------------------
def test_one_call_with_infinite_samples(sf, oracle, ctx):
    n = 2_000_000
    iq = synth_fsk(n, sps=100, seed=31, gap_every=100_000)   # unit amplitude plus noise: both parts of every sample are nonzero
    rng = np.random.default_rng(34)
    at = np.sort(rng.choice(np.arange(2, n - 2, 5), 100, replace=False))
    iq[at, 0] = rng.uniform(-1, 1, 100).astype(np.float32)
    iq[at, 1] = np.where(rng.random(100) < 0.5, INF, -INF).astype(np.float32)
    assert np.all(iq[at - 1] != 0) and np.all(iq[at + 1] != 0) and np.all(iq[at, 0] != 0)
    q_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert np.isfinite(q_ref).all()   # the recovery: a finite angle for the sample and for the one after it
    _check_center(sf, oracle, ctx, iq, 0.05, "FSK", tol=5, sps=100)
