"""CPU model of detect_center's binning in center.cu, pinned to numpy.

Restated here: the bin edges as np.arange forms them and as cen_edge forms them for k_center_plan and for caller-given edges
(one rounded product, one rounded sum; np.arange's length ceil((stop - start) / step)), the float thresholds ru(edge_k), rd(last edge) and
f_min = max(ru(hmin), succ(-4)), and HistBins::bin_of in both variants.  The FAST guess's FFMA is evaluated exactly
(fractions.Fraction) and rounded once to float32, so the model says what the device computes, not what float64 numpy would.
Pinned to np.histogram / np.searchsorted over many (hmin, hstep, nbins), with |edge| / hstep from 1 to past 2^24: the FAST guess
is never off by more than the one bin its look-up corrects while |edge| / hstep < 2^20 (the host's and k_center_plan's
condition), and beyond it the guess does go wrong, so the bound is needed."""
from fractions import Fraction

import numpy as np

F32 = np.float32
FAST_BOUND = 2.0 ** 20
SUCC_M4 = np.nextafter(F32(-4.0), F32(0.0))


def ru(x):
    """smallest float32 >= x (x: a Python / float64 number)"""
    f = F32(x)
    return np.nextafter(f, F32(np.inf)) if float(f) < x else f


def rd(x):
    f = F32(x)
    return np.nextafter(f, F32(-np.inf)) if float(f) > x else f


def f32_round(q: Fraction):
    """q rounded once to the nearest float32, ties to even (finite results only)"""
    if q == 0:
        return F32(0.0)
    sign = -1 if q < 0 else 1
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = a / ulp
    r = m.numerator // m.denominator
    rem = m - r
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and r % 2 == 1):
        r += 1
    return F32(sign * float(r * ulp))


def fmaf(a, b, c):
    return f32_round(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def arange_edges(hmin, hstep, nbins):
    """caller-given edges hmin + k * hstep, one rounded product and one rounded sum (np.arange's element formula)"""
    return hmin + np.arange(nbins + 1, dtype=np.float64) * hstep


def cen_edges(hmin, edge1, delta, nedges):
    """cen_edge: start, start + step, then start + k * delta"""
    e = hmin + np.arange(nedges, dtype=np.float64) * delta
    e[0] = hmin
    if nedges > 1:
        e[1] = edge1
    return e


class Bins:
    """the thresholds cen_edge_table writes and HistBins::load / bin_of reads"""

    def __init__(self, hmin, hstep, nbins):
        self.edges = arange_edges(hmin, hstep, nbins)
        self.nbins = nbins
        self.fe = np.array([ru(e) for e in self.edges], dtype=F32)
        self.f_hi = rd(self.edges[-1])
        self.f_min = max(ru(hmin), SUCC_M4)
        self.scale = F32(1.0 / hstep)
        self.off = -(self.fe[0] * self.scale)   # float32 product, negated
        self.ratio = max(abs(hmin), abs(self.edges[-1])) / hstep

    def valid(self, f):
        return bool(f >= self.f_min and f <= self.f_hi)

    def guess(self, f):
        """the FAST guess r before clamping: rn(fmaf(f, scale, off)) by the 1.5 * 2^23 trick"""
        t = fmaf(f, self.scale, self.off)
        with np.errstate(over="ignore"):
            s = F32(t + F32(12582912.0))
        return int(np.array(s, dtype=F32).view(np.int32)) - 0x4B400000

    def bin_fast(self, f):
        r = min(max(self.guess(f), 0), self.nbins)
        k = min(r - (1 if f < self.fe[r] else 0), self.nbins - 1)
        return k if self.valid(f) else -1

    def bin_loop(self, f):
        if not self.valid(f):
            return -1
        k = int((f - self.fe[0]) * self.scale)   # float32 difference and product, truncated
        k = max(0, min(k, self.nbins - 1))
        while k > 0 and f < self.fe[k]:
            k -= 1
        while k < self.nbins - 1 and f >= self.fe[k + 1]:
            k += 1
        return k


def reference_bin(f, edges):
    """np.histogram's bin of one float32 sample on the double edges (right-open bins, the last closed), -1 outside or not kept"""
    if not f > -4.0:
        return -1
    a = float(f)
    if not (edges[0] <= a <= edges[-1]):
        return -1
    return min(int(np.searchsorted(edges, a, side="right")) - 1, len(edges) - 2)


def probes(b: Bins, rng, n_random=60, exhaustive_bins=()):
    """samples on and next to every threshold kind, random samples over a wider range, and every float32 of some bins"""
    ks = sorted({0, 1, b.nbins // 2, b.nbins - 1, b.nbins} | set(rng.integers(0, b.nbins + 1, 6).tolist()))
    out = []
    for t in [b.fe[k] for k in ks] + [b.f_hi, b.f_min, F32(-4.0), SUCC_M4]:
        out += [t, np.nextafter(t, F32(-np.inf)), np.nextafter(t, F32(np.inf))]
    span = b.edges[-1] - b.edges[0]
    out += [F32(v) for v in rng.uniform(b.edges[0] - 0.02 * span, b.edges[-1] + 0.02 * span, n_random)]
    for k in exhaustive_bins:
        f = b.fe[k]
        while f <= b.fe[k + 1]:
            out.append(f)
            f = np.nextafter(f, F32(np.inf))
    return [F32(v) for v in out if np.isfinite(v)]


def _triples(rng):
    """(hmin, hstep, nbins) with |edge| / hstep from ~1 to 2^25, both signs, hmin around -4"""
    for nbins in (1, 2, 3, 7, 100, 1000, 6000):
        for log_ratio in np.linspace(0, 25, 26):
            hstep = float(10 ** rng.uniform(-4, 1))
            mag = max(2.0 ** log_ratio * hstep, nbins * hstep)
            hmin = float(rng.choice([-1, 1])) * mag - (nbins * hstep if rng.random() < 0.5 else 0.0)
            yield hmin, hstep, nbins
    yield -4.5, 0.25, 20          # f_min = succ(-4) cuts the first bins
    yield -4.0, 0.5, 10           # hmin == -4: the first edge is dropped by the keep rule
    yield float(np.float32(-3.9999998)), 1e-3, 500


def test_fast_guess_within_half_a_bin_under_the_bound():
    """below 2^20 the FAST guess is the true bin or the one above it, and bin_of<FAST> equals np.histogram's bin; the
    loop-based variant equals it everywhere"""
    rng = np.random.default_rng(2024)
    checked_fast = worst = 0
    for hmin, hstep, nbins in _triples(rng):
        b = Bins(hmin, hstep, nbins)
        for f in probes(b, rng):
            want = reference_bin(f, b.edges)
            assert b.bin_loop(f) == want, (hmin, hstep, nbins, f)
            if b.ratio < FAST_BOUND and want >= 0:
                r = min(max(b.guess(f), 0), nbins)
                assert r - want in (0, 1), (hmin, hstep, nbins, f, r, want)
                assert b.bin_fast(f) == want, (hmin, hstep, nbins, f)
                checked_fast += 1
                worst = max(worst, b.ratio)
            elif b.ratio < FAST_BOUND:
                assert b.bin_fast(f) == -1
    assert checked_fast > 5000 and worst > FAST_BOUND / 2


def test_exhaustive_bins_next_to_the_fast_bound():
    """every float32 of the first, middle and last bins of ranges whose |edge| / hstep lies just below 2^20, one with hmin just
    above a float32 (ru(hmin) almost an ulp above it, the guess's worst start)"""
    rng = np.random.default_rng(7)
    for hmin, nbins in ((1000.0, 200), (-1000.0, 200), (1000.0 + 0.01 * 2.0 ** -14, 200), (4999.5, 6000), (-3.9, 50)):
        hstep = abs(hmin) / (FAST_BOUND - nbins - 8)
        b = Bins(hmin, hstep, nbins)
        assert FAST_BOUND * 0.99 < b.ratio < FAST_BOUND
        samples = probes(b, rng, 0, exhaustive_bins=(0, 1, nbins // 2, nbins - 2, nbins - 1))
        assert len(samples) > 40
        for f in samples:
            want = reference_bin(f, b.edges)
            assert b.bin_fast(f) == want, (hmin, hstep, f)
            assert b.bin_loop(f) == want, (hmin, hstep, f)


def test_fast_guess_fails_past_the_bound():
    """the bound is needed: between 2^21 and 2^25 the one-look-up guess misses bins the loop finds.  The guess counts from
    ru(hmin), which lies up to an ulp above hmin: an ulp of hmin is ratio * 2^-23 bins, so past 2^20 the guess can be a bin low."""
    rng = np.random.default_rng(99)
    missed = 0
    between = 30000.0 + 0.01 * 2.0 ** -9   # just above a float32
    b = Bins(between, between / 2 ** 23.5, 3000)
    assert b.ratio < 2 ** 24 and any(b.bin_fast(f) != reference_bin(f, b.edges) for f in probes(b, rng, 300))
    for hmin, nbins in ((3.0e4, 3000), (-3.0e4, 3000), (5.0e6, 500)):
        for ratio in (2.0 ** 22, 2.0 ** 23.5, 2.0 ** 24.5):
            hstep = abs(hmin) / ratio
            b = Bins(hmin, hstep, nbins)
            for f in probes(b, rng, 200):
                want = reference_bin(f, b.edges)
                assert b.bin_loop(f) == want
                missed += b.bin_fast(f) != want
    assert missed > 0


def test_f32_round_is_round_to_nearest_even():
    rng = np.random.default_rng(3)
    for _ in range(2000):
        a = float(rng.standard_normal() * 10 ** rng.uniform(-30, 30))
        assert f32_round(Fraction(a)) == F32(a)   # float64 -> float32 rounds once, to nearest even
    one = Fraction(1)
    half_ulp = Fraction(1, 2 ** 24)
    assert f32_round(one + half_ulp) == F32(1.0)                       # tie to even
    assert f32_round(one + 3 * half_ulp) == F32(1.0) + F32(2.0 ** -22)   # tie to even, upwards
    assert f32_round(one + half_ulp + Fraction(1, 2 ** 80)) == np.nextafter(F32(1.0), F32(2.0))


def plan_edges(mn, mx, var):
    """k_center_plan's restatement of np.arange(mn, mx + var, var): length ceil((stop - start) / step), elements start,
    start + step, then start + k * delta with delta = (start + step) - start; None where it records no histogram"""
    hstep = float(np.float32(var))
    if hstep == 0.0:
        return None
    stop = mx + hstep
    val = (stop - mn) / hstep
    if not (val == val and abs(val) < 9.0e18):
        return None
    length = int(np.ceil(val))
    if length < 2:
        return None
    edge1 = mn + hstep
    return cen_edges(mn, edge1, edge1 - mn, length)


def test_plan_edges_are_np_arange():
    """k_center_plan's edges equal np.arange's, bit for bit, at random windows and where the length sits on a ceil boundary"""
    rng = np.random.default_rng(11)
    cases = []
    for _ in range(3000):
        mn = float(np.float32(rng.uniform(-4, 4) * 10 ** rng.uniform(-3, 4)))
        var = float(np.float32(10 ** rng.uniform(-6, 1) * max(1.0, abs(mn)) ** rng.uniform(0, 1)))
        nb = int(rng.integers(1, 7000))
        mx = float(np.float32(mn + var * (nb + rng.choice([-1e-7, 0.0, 1e-7, 0.5]))))
        cases.append((mn, mx, var))
    # exact lengths: max - min a whole number of steps (dyadic steps), one edge, 6000 and 6001 bins
    for nb in (0, 1, 2, 5999, 6000, 6001):
        for var in (0.25, 2.0 ** -10, 0.125):
            cases.append((-1.0, -1.0 + nb * var, var))
    hit_exact = 0
    for mn, mx, var in cases:
        want = np.arange(mn, mx + float(np.float32(var)), float(np.float32(var)))
        got = plan_edges(mn, mx, var)
        if len(want) < 2:
            assert got is None, (mn, mx, var)
            continue
        assert got is not None and np.array_equal(got.view(np.uint64), want.view(np.uint64)), (mn, mx, var)
        hit_exact += float(np.ceil((mx + np.float32(var) - mn) / np.float32(var))) == (mx + np.float32(var) - mn) / np.float32(var)
    assert hit_exact >= 10

