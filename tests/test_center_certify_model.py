"""numpy restatement of the certified peak pick (center.cu k_center_certify, DESIGN.md §4.4.1), no GPU.

The demodulation pass counts the kept samples into a fine histogram of fixed buckets; for every bin of detect_center's histogram
the certificate derives L_k <= count_k <= U_k from the buckets (plus exact counts of the samples that were not bucketed) and
decides the two peaks only when every count vector within the bounds gives the same two.  Checked here: the bounds hold on
random captures and near-ties, a certified center equals detect_center (oracle.py, the reference's numpy code restated), and a
cluster split evenly by a bin edge is refused."""
import numpy as np

from test_hist_binning_model import rd, ru

NB = 4096
GRID = {"FSK": (np.float32(512.0), np.float32(2048.0)), "ASK": (np.float32(4096.0), np.float32(0.0))}


def bucket(f, scale, off):
    """urh_fine_bucket: floor(f * scale) + off clamped to [0, NB) (f * scale is exact in float64: the scale is a power of two)"""
    with np.errstate(invalid="ignore"):
        b = np.floor(np.asarray(f, np.float32).astype(np.float64) * float(scale)) + float(off)
    return np.clip(np.nan_to_num(b, nan=0.0, posinf=NB - 1, neginf=0), 0, NB - 1).astype(np.int64)


def thresholds(hmin, hstep, nbins):
    """k_center_plan: fe[0..nbins] = ru(edge_k), f_hi = rd(last edge), f_min = max(ru(hmin), pred(-4) toward 0)"""
    k = np.arange(nbins + 1, dtype=np.float64)
    edges = hmin + k * hstep
    edges[1] = hmin + hstep
    fe = ru(edges)
    return fe, rd(edges[-1:])[0], max(ru(np.array([hmin]))[0], np.nextafter(np.float32(-4), np.float32(0)))


def exact_counts(v, fe, f_hi, f_min):
    """HistBins::bin_of over float32 values v"""
    v = v[(v >= f_min) & (v <= f_hi)]
    k = np.searchsorted(fe, v, side="right") - 1
    return np.bincount(np.minimum(k, len(fe) - 2), minlength=len(fe) - 1)


def bounds(bucketed, exact, fe, f_hi, f_min, scale, off):
    """L_k, U_k of every bin from the bucket counts of `bucketed` (kept float32 samples) plus the exact counts `exact`"""
    B = np.bincount(bucket(bucketed, scale, off), minlength=NB).astype(np.int64)
    ge = np.concatenate([np.cumsum(B[::-1])[::-1], [0]])   # ge[b] = samples in buckets >= b

    def g(t):
        bt = bucket(t, scale, off)
        straddles = bucket(np.nextafter(t, np.float32(-np.inf)), scale, off) == bt
        return np.where(straddles, ge[bt + 1], ge[bt]), ge[bt]

    nbins = len(fe) - 1
    top = np.nextafter(np.float32(f_hi), np.float32(np.inf))
    a = np.maximum(fe[:-1], f_min)
    e = np.minimum(fe[1:], top)
    e[-1] = top
    alo, ahi = g(a)
    elo, ehi = g(e)
    nonempty = a < e
    L = np.where(nonempty, np.maximum(alo - ehi, 0), 0) + exact
    U = np.where(nonempty, ahi - elo, 0) + exact
    assert len(L) == nbins
    return L, U


def certify(L, U):
    """the two bins that are peaks for every count vector within [L, U] and exceed every other possible peak, or None"""
    n = len(L)
    w = max(2, int(0.05 * n) + 1)
    certain, possible = [], []
    for k in range(n):
        nb = [j for j in range(k - w + 1, k + w) if j != k and 0 <= j < n]
        if L[k] > 0 and all(L[k] > U[j] for j in nb):
            certain.append(k)
        if U[k] > 0 and all(U[k] > L[j] for j in nb):
            possible.append(k)
    if len(certain) < 2:
        return None
    k1, k2 = sorted(certain, key=lambda k: (-L[k], k))[:2]
    rest = [U[j] for j in possible if j not in (k1, k2)]
    return (k1, k2) if L[k2] > max(rest, default=0) else None


def window(q, max_size=None):
    rect = q[q > -4]
    rect = rect[int(0.05 * len(rect)): int(0.95 * len(rect))]
    if max_size is not None and len(rect) > max_size:
        rect = rect[:max_size]
    return rect


def plan(rect):
    hmin, hstep = float(rect.min()), float(np.var(rect))
    nbins = len(np.arange(hmin, float(rect.max()) + hstep, hstep)) - 1
    return hmin, hstep, nbins


def fsk_qad(n, seed, dev=0.314, sigma=0.014, noise_frac=0.2):
    rng = np.random.default_rng(seed)
    q = np.where(rng.integers(0, 2, n // 100 + 1).repeat(100)[:n] > 0, dev, -dev) + sigma * rng.standard_normal(n)
    q[rng.random(n) < 0.001] = rng.uniform(-np.pi, np.pi)          # burst starts: random phase
    q[rng.random(n) < noise_frac] = -4.0                             # gated samples
    return q.astype(np.float32)


def model_center(q, mod="FSK", exact_frac=0.05, seed=0, max_size=None):
    """certified center of q or None; the samples of a random contiguous run in the window are bucketed, the rest counted
    exactly (the slabs wholly inside the window vs the cut slabs); asserts the bounds on the way"""
    rect = window(q, max_size)
    hmin, hstep, nbins = plan(rect)
    if not (hstep > 0 and 2 <= nbins + 1 and nbins <= 6000):
        return None, None
    fe, f_hi, f_min = thresholds(hmin, hstep, nbins)
    rng = np.random.default_rng(seed)
    m = len(rect)
    a = int(rng.integers(0, max(1, int(exact_frac * m)) + 1))
    b = m - int(rng.integers(0, max(1, int(exact_frac * m)) + 1))
    exact = exact_counts(rect[:a], fe, f_hi, f_min) + exact_counts(rect[b:], fe, f_hi, f_min)
    L, U = bounds(rect[a:b], exact, fe, f_hi, f_min, *GRID[mod])
    truth = exact_counts(rect, fe, f_hi, f_min)
    ref, _ = np.histogram(rect, bins=np.arange(hmin, float(rect.max()) + hstep, hstep))
    assert np.array_equal(truth, ref)
    assert (L <= truth).all() and (truth <= U).all()
    pick = certify(L, U)
    if pick is None:
        return None, truth
    edges = np.arange(hmin, float(rect.max()) + hstep, hstep)
    return float(np.mean([edges[pick[0]], edges[pick[1]]])), truth


def test_bucket_is_monotone():
    rng = np.random.default_rng(1)
    for mod, (scale, off) in GRID.items():
        f = np.sort(np.concatenate([rng.uniform(-5, 5, 200_000), rng.uniform(-1e-6, 1e-6, 1000)]).astype(np.float32))
        f = np.concatenate([f, np.float32([np.inf])])
        assert (np.diff(bucket(f, scale, off)) >= 0).all(), mod


def test_bounds_and_certified_center_match_detect_center():
    from oracle import oracle

    certified = 0
    for seed in range(12):
        q = fsk_qad(200_000 + 7919 * seed, seed)
        for max_size in (None, 50_000):
            c, _ = model_center(q, "FSK", seed=seed, max_size=max_size)
            if c is not None:
                certified += 1
                assert c == oracle.detect_center(q, max_size)
    assert certified >= 20


def test_ask_levels():
    from oracle import oracle

    rng = np.random.default_rng(5)
    n = 300_000
    q = (np.where(rng.integers(0, 2, n // 100 + 1).repeat(100)[:n] > 0, 0.8, 0.3) + 0.01 * rng.standard_normal(n)).astype(np.float32)
    q[rng.random(n) < 0.1] = -4.0
    c, _ = model_center(q, "ASK", seed=5)
    assert c is not None and c == oracle.detect_center(q)


def test_bounds_hold_on_near_ties():
    """three clusters whose populations differ by a few samples: the bounds hold, and whatever is certified is detect_center's
    answer"""
    from oracle import oracle

    rng = np.random.default_rng(9)
    for trial in range(30):
        n = 40_000
        levels = rng.uniform(-1, 1, 3)
        counts = n // 3 + rng.integers(-3, 4, 3)
        q = np.concatenate([np.full(c, lv, np.float32) + np.float32(1e-4) * rng.standard_normal(c).astype(np.float32)
                            for lv, c in zip(levels, counts)])
        q = q[rng.permutation(len(q))]
        c, _ = model_center(q, "FSK", seed=trial)
        if c is not None:
            assert c == oracle.detect_center(q)


def test_even_split_of_a_cluster_is_refused():
    """a cluster that a bin edge splits evenly inside one bucket: neither half is a certain peak, and the bucket could make
    either bin a peak above the second cluster - the certificate must refuse"""
    hmin, hstep, nbins = -1.0, 0.1, 20
    fe, f_hi, f_min = thresholds(hmin, hstep, nbins)
    t = fe[12]
    big = np.full(1000, np.float32(-0.55))
    second = np.full(300, np.float32(0.65))
    split = np.concatenate([np.full(500, np.nextafter(t, np.float32(-1))), np.full(500, t)]).astype(np.float32)
    assert bucket(split[:1], *GRID["FSK"])[0] == bucket(split[-1:], *GRID["FSK"])[0]
    v = np.concatenate([big, second, split, np.float32([hmin, hmin + nbins * hstep - 1e-3])])
    truth = exact_counts(v, fe, f_hi, f_min)
    L, U = bounds(v, np.zeros(nbins, np.int64), fe, f_hi, f_min, *GRID["FSK"])
    assert (L <= truth).all() and (truth <= U).all()
    assert L[11] == 0 and L[12] == 0 and U[11] >= 500 and U[12] >= 500
    assert certify(L, U) is None
    # counted exactly instead, the same samples certify: the refusal comes from the straddling bucket alone
    assert certify(truth, truth) is not None
