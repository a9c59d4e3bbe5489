"""Complex64 (x, taps) pairs at the edges of fir_filter (signal_functions.pyx:513-525), each with a name and a group.

tests/test_oracle.py pins the oracle's fir_filter to the reference's on them (recorded in tests/golden/ref_fir_edges.json);
tests/test_gpu_fir_edges.py runs them through every device FIR entry point against the oracle.  The reference adds
x[i] * taps[k - i] over its real samples, i ascending, to an output that starts at +0, each product std::complex<float>'s
(libgcc's __mulsc3: the naive product, with C99 Annex G's recovery when both parts are NaN).  The groups:
* shapes: m in {1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025, 4001} against n in {1, 2, m - 1, m, m + 1, 1023, 1024, 1025, 2047,
  2049, 3 * 1024 + 1} (1024 outputs per block, 4 per thread); odd and even m and n decide which blocks take the bulk tile copy;
* nonfinite_samples: +-inf, NaN and their mixes in either part, at sample 0, the last sample, 1023, 1024, the first and last
  sample of the halo the tile at 2048 reads, and inside the first m - 1 outputs, with real and complex taps;
* nonfinite_taps: real inf, imaginary inf, both, NaN in either part, at q = 0, m // 2 and m - 1 (q > k pairs a tap with the zero
  initial state for output k, which the reference never multiplies), n > m and n < m;
* annexg: the three recovery branches of __mulsc3: an infinite sample, an infinite tap, and finite operands whose partial products
  overflow while a NaN is present, plus the examples of the products the recovery changes;
* overflow: sums that overflow to +inf and then meet -inf (NaN in both parts without any NaN product);
* subnormal: products in the subnormal range, sums of subnormal samples and taps, results next to FLT_MIN (no flush to zero);
* signed_zero: -0 samples and taps, outputs all of whose terms are -0 (the reference's output is +0: np.zeros start);
* large_m: 12287 taps (the last count whose tile fits in shared memory), 12288 and 20000, n <= 5000, and one capture longer
  than its 12288 taps (a second shard's history);
* empty: no taps (n - 1 outputs; n = 0 raises ValueError) and no samples."""
import numpy as np

F = np.float32
C64 = np.complex64
TILE = 1024
INF, NAN = float("inf"), float("nan")
FLT_MIN = float(np.finfo(np.float32).tiny)

# (real, imaginary) of every non-finite sample kind
NONFINITE = [(INF, 0.0), (-INF, 0.0), (0.0, INF), (0.0, -INF), (INF, INF), (INF, -INF), (NAN, 0.0), (0.0, NAN), (NAN, NAN),
             (INF, NAN), (NAN, -INF), (-INF, 2.0)]
NONFINITE_TAPS = [(INF, 0.0), (-INF, 0.0), (0.0, INF), (INF, INF), (NAN, 0.0), (0.0, NAN), (NAN, NAN)]
SHAPE_M = [1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025, 4001]


class Case:
    __slots__ = ("name", "group", "x", "taps")

    def __init__(self, name, group, x, taps):
        self.name, self.group = name, group
        self.x, self.taps = c64(x), c64(taps)


def c64(v):
    """a complex64 array; (re, im) pairs are taken word for word (complex() would turn inf * 1j into nan + inf j)"""
    if isinstance(v, np.ndarray):
        return np.ascontiguousarray(v, dtype=C64)
    pairs = [p if isinstance(p, tuple) else (complex(p).real, complex(p).imag) for p in v]
    return np.ascontiguousarray(np.array(pairs, dtype=F).reshape(-1, 2)).view(C64).ravel()


def _noise(n, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * scale).astype(C64)


def _taps(m, seed, real=False):
    rng = np.random.default_rng(10_000 + seed)
    t = rng.standard_normal(m) + (0 if real else 1j * rng.standard_normal(m))
    return (t / np.sqrt(max(m, 1))).astype(C64)


def folded(y):
    """the float32 words of a complex64 result, every NaN folded to 0x7fc00000 (the payload is not pinned); -0 and +0 stay apart"""
    f = np.ascontiguousarray(y, dtype=C64).view(F)
    w = f.view(np.uint32).copy()
    w[np.isnan(f)] = 0x7FC00000
    return w


def fast_loop(x, taps):
    """k_fir_exact's tap loop restated: every output starts at +0 and adds x[k - q] * taps[q] for q = m - 1 .. 0, the samples
    before x[0] being 0, with the naive product (no Annex G recovery).  The reference differs from it exactly where the kernel
    needs its recheck."""
    x, taps = c64(x), c64(taps)
    n, m = len(x), len(taps)
    xr = np.concatenate([np.zeros(max(m - 1, 0), F), x.real.astype(F)])
    xi = np.concatenate([np.zeros(max(m - 1, 0), F), x.imag.astype(F)])
    re, im = np.zeros(n, F), np.zeros(n, F)
    with np.errstate(all="ignore"):
        for q in range(m - 1, -1, -1):
            vr, vi = xr[m - 1 - q: m - 1 - q + n], xi[m - 1 - q: m - 1 - q + n]
            hr, hi = F(taps[q].real), F(taps[q].imag)
            re = re + ((vr * hr) - (vi * hi))
            im = im + ((vr * hi) + (vi * hr))
    return np.ascontiguousarray(np.stack([re, im], 1)).view(C64).ravel()


def cases():
    """every Case, names unique"""
    with np.errstate(over="ignore", invalid="ignore"):   # scaled noise may overflow to inf: those samples are cases too
        return _cases()


def _cases():
    out = []

    def add(name, group, x, taps):
        out.append(Case(name, group, x, taps))

    # ---- shapes -------------------------------------------------------------------------------------------------------------------
    for m in SHAPE_M:
        for n in sorted({1, 2, m - 1, m, m + 1, 1023, 1024, 1025, 2047, 2049, 3 * TILE + 1} - {0}):
            add("shape_m%d_n%d" % (m, n), "shapes", _noise(n, 7 * m + n), _taps(m, m + n, real=(n % 3 == 0)))

    # ---- non-finite samples ---------------------------------------------------------------------------------------------------------
    n = 3 * TILE + 1
    for m in (3, 4, 33, 1025):
        where = {"first": 0, "last": n - 1, "at1023": 1023, "at1024": 1024, "halo_lo": 2 * TILE - (m - 1), "halo_hi": 2 * TILE - 1,
                 "head": (m - 1) // 2}
        for j, v in enumerate(NONFINITE):
            for pos, p in where.items():
                x = _noise(n, 100 * m + j)
                x[p] = c64([v])[0]
                add("sample_%s_%s_m%d_v%d" % (pos, "real" if j % 2 else "cplx", m, j), "nonfinite_samples", x, _taps(m, j, real=j % 2 == 1))
        # every kind at once, a few samples apart: infinities of both signs meet in one sum
        x = _noise(n, 5 * m)
        rng = np.random.default_rng(m)
        for p in rng.choice(n, 60, replace=False):
            x[p] = c64([NONFINITE[p % len(NONFINITE)]])[0]
        add("sample_mixed_m%d" % m, "nonfinite_samples", x, _taps(m, 3, real=m % 2 == 1))

    # ---- non-finite taps -------------------------------------------------------------------------------------------------------------
    for m in (1, 2, 3, 5, 33, 1025):
        for j, v in enumerate(NONFINITE_TAPS):
            for q in sorted({0, m // 2, m - 1}):
                for n in ((3 * TILE + 1, m - 1) if m >= 3 else (3 * TILE + 1,)):
                    t = _taps(m, 20 * m + j, real=j % 2 == 0)
                    t[q] = c64([v])[0]
                    add("tap_q%d_m%d_v%d_n%d" % (q, m, j, n), "nonfinite_taps", _noise(n, 300 + m + j), t)

    # ---- the three branches of __mulsc3's recovery, and the examples ------------------------------------------------------------------
    add("annexg_inf_sample_example", "annexg", [(1, 1), (INF, INF), (2, 0), (3, 0)], [0.1, 0.2, 0.3])
    add("annexg_inf_nan_sample", "annexg", [(INF, NAN)], [1.0])
    add("annexg_overflow_nan_example", "annexg", [(NAN, 1e30)], [(1e30, 1e30)])
    add("annexg_padded_inf_tap_example", "annexg", [(1, 1), (2, 0), (3, 0)], [1.0, INF])
    add("annexg_padded_inf_tap3_example", "annexg", [(1, 1), (2, 0), (3, 0)], [0.5, 0.25, INF])
    x = _noise(2 * TILE + 5, 41)
    x[[5, 700, 1023, 1500]] = c64([(INF, INF), (-INF, -INF), (INF, -INF), (-INF, 0.5)])
    add("annexg_inf_samples_real_taps", "annexg", x, _taps(5, 41, real=True))
    t = _taps(6, 42, real=True)
    t[[1, 4]] = c64([(INF, 0.0), (-INF, -INF)])
    add("annexg_inf_taps", "annexg", np.abs(_noise(2 * TILE + 5, 42)).astype(C64), t)   # real samples: (inf, 0) * (a, 0) recovers
    # finite operands, partial products overflow, a NaN in one part: the third branch
    big = _noise(TILE + 7, 43, 1e30)
    big[3::11] = c64([(NAN, 1e30)])[0]
    big[8::13] = c64([(2e30, NAN)])[0]
    add("annexg_overflow_nan_samples", "annexg", big, _taps(3, 43) * C64(1e30))
    t = _taps(4, 44) * C64(1e30)
    t[2] = c64([(NAN, 3e30)])[0]
    add("annexg_overflow_nan_tap", "annexg", _noise(TILE + 9, 44, 1e25), t)

    # ---- sums that overflow and meet -inf ---------------------------------------------------------------------------------------------
    add("overflow_then_neginf_real", "overflow", [(3e38, 0), (3e38, 0), (3e38, 0), (-INF, 0), (3e38, 0), (1, 0), (2, 0)], [1.0, 1.0, 1.0])
    add("overflow_then_neginf_imag", "overflow", [(0, 3e38), (0, 3e38), (0, 3e38), (0, -INF), (0, 3e38), (0, 1), (0, 2)], [1.0, 1.0, 1.0])
    x = _noise(2 * TILE + 3, 51) * C64(1e38)
    x[[100, 1030, 2000]] = c64([(-INF, -INF), (-INF, 0.0), (0.0, -INF)])
    add("overflow_wide_neginf", "overflow", x, np.full(7, 1.5 + 1.5j, C64))
    add("overflow_alternating", "overflow", np.tile(c64([(3e38, -3e38), (3e38, -3e38), (-3e38, 3e38)]), 400), [2.0, (1 + 1j), 2.0, 1.0])

    # ---- subnormals -------------------------------------------------------------------------------------------------------------------
    add("subnormal_products", "subnormal", _noise(TILE + 5, 61, 1e-20), _taps(5, 61) * C64(1e-20))
    add("subnormal_samples", "subnormal", _noise(TILE + 5, 62, 1e-39), _taps(4, 62))
    add("subnormal_taps", "subnormal", _noise(TILE + 5, 63), _taps(33, 63) * C64(1e-39))
    rng = np.random.default_rng(64)
    near = (FLT_MIN * rng.uniform(0.4, 1.2, TILE + 5) + 1j * FLT_MIN * rng.uniform(-1.2, 1.2, TILE + 5)).astype(C64)
    add("subnormal_near_flt_min", "subnormal", near, [0.5, 0.25, 0.75, (0.5, 0.5), 1.0])
    add("subnormal_tiny_sums", "subnormal", np.full(TILE + 5, 1e-45 + 1e-45j, C64), np.full(9, 1.5 + 0.5j, C64))

    # ---- signed zeros -----------------------------------------------------------------------------------------------------------------
    add("neg_zero_samples", "signed_zero", np.full(TILE + 3, complex(-0.0, -0.0), C64), _taps(5, 71))
    add("neg_zero_taps", "signed_zero", _noise(TILE + 3, 72), c64([(-0.0, -0.0)] * 4))
    # every term -0 in both parts: (-0 + 0j) * (1 + 0j) = (-0 - 0, -0 + 0) and (-0 - 0j) * (1 + 0j) = (-0 + 0, -0 - 0) ... the output
    # is +0 because the reference starts from +0
    add("neg_zero_all_terms", "signed_zero", np.tile(c64([(-0.0, 0.0), (-0.0, -0.0), (0.0, -0.0)]), 350), c64([(1.0, 0.0), (1.0, -0.0), (-0.0, -1.0)]))
    rng = np.random.default_rng(73)
    x = c64(np.stack([rng.choice([0.0, -0.0, 1.0, -1.0], 2 * TILE + 1), rng.choice([0.0, -0.0, 1.0, -1.0], 2 * TILE + 1)], 1).astype(F)
            .view(C64).ravel())
    add("signed_zero_mixed", "signed_zero", x, c64([(-0.0, 0.0), (1.0, -0.0), (0.0, 0.0), (-1.0, -0.0), (-0.0, -0.0)]))

    # ---- tap counts past the shared-memory tile ---------------------------------------------------------------------------------------
    for m, n in ((12287, 5000), (12287, 2049), (12288, 5000), (12288, 1), (12288, 1025), (20000, 4097), (20000, 5000)):
        add("large_m%d_n%d" % (m, n), "large_m", _noise(n, m + n), _taps(m, m + n, real=(n % 2 == 1)))
    x = _noise(5000, 81)
    x[3000] = c64([(INF, INF)])[0]
    x[4500] = c64([(NAN, 0.0)])[0]
    add("large_m20000_nonfinite_samples", "large_m", x, _taps(20000, 81, real=True))
    t = _taps(12288, 82)
    t[[0, 6000, 12287]] = c64([(INF, 0.0), (NAN, 0.0), (0.0, -INF)])
    add("large_m12288_nonfinite_taps", "large_m", _noise(4097, 82), t)
    # longer than the taps, so that a second shard can take its m - 1 samples of history from the first
    x = _noise(12288 + 1025, 83)
    x[13000] = c64([(INF, INF)])[0]
    add("large_m12288_n13313_history", "large_m", x, _taps(12288, 83, real=True))

    # ---- empty inputs -----------------------------------------------------------------------------------------------------------------
    for n in (0, 1, 3):
        add("empty_taps_n%d" % n, "empty", _noise(n, 90 + n), np.zeros(0, C64))
    add("empty_samples_m2", "empty", np.zeros(0, C64), _taps(2, 93))
    add("empty_samples_m1", "empty", np.zeros(0, C64), _taps(1, 94))

    names = [c.name for c in out]
    assert len(names) == len(set(names)), "case names must be unique"
    return out


GROUPS = ["shapes", "nonfinite_samples", "nonfinite_taps", "annexg", "overflow", "subnormal", "signed_zero", "large_m", "empty"]
