"""CPU model of the speculative digitizer's proof (UrhSpec, DESIGN.md §4.4.1), in float32 as the kernels compute it.

A tile digitized at the guess t_g keeps its classes at the detected threshold c when min over the tile of fl(|s - t_g|) exceeds
fl(|c - t_g|): a sample whose class differs between the two thresholds lies in (t_g, c] or (c, t_g], and round-to-nearest is
monotone, so its fl(|s - t_g|) cannot exceed fl(|c - t_g|).  Whenever the inequality holds, (s > t_g) == (s > c) for every sample,
gated samples (the -4 sentinel) included."""
import numpy as np

F = np.float32
PI = F(np.pi)
SPECIAL = np.array([0.0, -0.0, PI, -PI, -4.0, np.nextafter(PI, F(0)), np.nextafter(-PI, F(0)), 1e-38, -1e-38, 1e-45, -1e-45],
                   dtype=F)


def _check(s, tg, c):
    s = np.asarray(s, dtype=F)
    tg, c = F(tg), F(c)
    margin = np.abs(s - tg).min()        # float32 subtraction, rounded to nearest
    if margin > np.abs(c - tg):
        assert np.array_equal(s > tg, s > c), (tg, c, s[(s > tg) != (s > c)])
        return True
    return False


def _neighbours(x, k=3):
    out = [F(x)]
    up = dn = F(x)
    for _ in range(k):
        up = np.nextafter(up, F(np.inf))
        dn = np.nextafter(dn, F(-np.inf))
        out += [up, dn]
    return out


def test_random_tiles():
    rng = np.random.default_rng(0)
    held = 0
    for _ in range(4000):
        tg = F(rng.uniform(-np.pi, np.pi))
        c = F(tg + rng.normal(0, 10.0 ** rng.uniform(-7, -1)))
        width = 10.0 ** rng.uniform(-7, 0.5)
        s = (rng.uniform(-1, 1, 256) * width + rng.choice([tg, c, -0.3, 0.3])).astype(F)
        s[rng.integers(0, 256, 8)] = -4.0
        held += _check(s, tg, c)
    assert held > 500


def test_samples_on_and_next_to_both_thresholds():
    rng = np.random.default_rng(1)
    held = 0
    for _ in range(3000):
        tg = F(rng.uniform(-np.pi, np.pi)) if rng.random() < 0.8 else rng.choice(SPECIAL)
        c = rng.choice(_neighbours(tg, 40)) if rng.random() < 0.5 else F(tg + rng.normal(0, 1e-3))
        pool = np.array(_neighbours(tg) + _neighbours(c) + list(SPECIAL), dtype=F)
        for _ in range(4):
            s = rng.choice(pool, size=rng.integers(1, 12))
            held += _check(s, tg, c)
            # each sample alone: the proof must hold sample by sample too
            for v in s:
                held += _check([v], tg, c)
    assert held > 1000


def test_ties_and_extremes():
    for tg in SPECIAL:
        for c in SPECIAL:
            for s in SPECIAL:
                _check([s], tg, c)
            _check(SPECIAL, tg, c)
    # |s - t_g| == |c - t_g| exactly (s mirrored about t_g, or s == c): never strictly greater, so never trusted
    assert not _check([F(0.5)], F(0.25), F(0.0))
    assert not _check([F(0.0)], F(0.25), F(0.0))
    assert _check([F(0.5), F(-4.0)], F(0.25), F(0.2))


def test_gated_sentinel_only_lowers_the_margin():
    s = np.array([0.3, -0.3, 0.31], dtype=F)
    tg, c = F(0.01), F(0.02)
    with_noise = np.append(s, F(-4.0))
    assert np.abs(with_noise - tg).min() <= np.abs(s - tg).min()
    assert _check(s, tg, c) and _check(with_noise, tg, c)
