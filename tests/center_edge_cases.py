"""Float32 "qad" arrays at the edges of detect_center (AutoInterpretation.py:226-277), each with a name.

tests/test_oracle.py pins the oracle's detect_center to the reference's on them (recorded in tests/golden/ref_center_edges.json);
tests/test_gpu_center_edges.py compares the device paths with the oracle.  They cover:
* the keep rule: exactly -4.0 (dropped), pred(-4) towards 0 (kept, the histogram's floor), -inf and NaN (dropped), +inf inside the
  rank window (np.arange raises, no center) and only in the trimmed 5 %;
* huge, subnormal, all-equal and bin-count-overflowing windows, windows of 0, 1, 2 and 3 kept samples;
* samples exactly on bin edges: levels whose variance is dyadic, integer-valued magnitudes;
* rank windows at tile (2048-sample) boundaries, inside one tile, over silent tiles, cut by max_size mid-tile;
* a level far from zero relative to its spread (|edge| / bin width near 2^20, and the nearly constant carrier whose variance
  cancels in Σx² - n·mean²).
Every case keeps np.arange's bin count at most ~10^6 or makes np.arange refuse the length outright."""
import numpy as np

TILE = 2048
M4 = np.float32(-4.0)
ABOVE_M4 = np.nextafter(np.float32(-4.0), np.float32(0.0))   # the smallest kept value


def _bimodal(n, seed, lo=-0.5, hi=0.5, sigma=0.05, run=40):
    rng = np.random.default_rng(seed)
    lv = np.repeat(np.where(rng.integers(0, 2, n // run + 1) > 0, hi, lo), run)[:n]
    return (lv + sigma * rng.standard_normal(n)).astype(np.float32)


def _put(x, idx, v):
    x = x.copy()
    x[np.asarray(idx) % len(x)] = v
    return x


def _kept_index(x, rank):
    """position of the kept sample of the given rank"""
    return int(np.nonzero(x > -4)[0][rank])


def cases():
    """(name, float32 array, max_size) for every case"""
    out = []

    def add(name, x, max_size=None):
        out.append((name, np.ascontiguousarray(x, dtype=np.float32), max_size))

    base = _bimodal(20_000, 1)
    add("bimodal", base)
    add("bimodal_max_size", base, 3000)
    # the keep rule
    add("minus4_exact", _put(base, np.arange(0, 20_000, 7), M4))
    add("minus4_and_floor", _put(_put(base, np.arange(0, 20_000, 7), M4), np.arange(3, 20_000, 997), ABOVE_M4))
    add("floor_only_kept_low", _put(_bimodal(5000, 2, lo=-3.5, hi=-3.0), np.arange(1, 5000, 50), ABOVE_M4))
    x = _put(base, np.arange(0, 20_000, 5), np.nan)
    add("nan_neginf", _put(x, np.arange(2, 20_000, 11), -np.inf))
    add("below_minus4", _put(base, np.arange(0, 20_000, 3), np.float32(-4.5)))
    add("posinf_in_window", _put(base, [10_000], np.inf))
    add("neg_huge_in_window", _put(base, [10_000], np.float32(-3.9)))
    x = base.copy()
    x[:100] = np.inf     # ranks 0..99 of 20000: inside the trimmed first 5 %
    x[-50:] = np.inf     # and the trimmed last 5 %
    add("posinf_trimmed", x)
    x = _put(base, np.arange(0, 20_000, 4), M4)   # 15000 kept; rank 749 is the last trimmed one
    x[_kept_index(x, 749)] = np.inf
    add("posinf_last_trimmed_rank", x)
    x = _put(base, np.arange(0, 20_000, 4), M4)
    x[_kept_index(x, 750)] = np.inf
    add("posinf_first_window_rank", x)
    # scale: huge, subnormal, all-equal, a bin count np.arange refuses
    fmax = np.finfo(np.float32).max
    add("flt_max_levels", np.where(base > 0, fmax, -fmax).astype(np.float32))
    add("huge_levels", (base * np.float32(1e18)).astype(np.float32))
    add("subnormal_levels", (base * np.float32(1e-39)).astype(np.float32))
    add("bins_overflow", (base * np.float32(1e-21)).astype(np.float32))
    add("all_equal", np.full(5000, 0.7, np.float32))
    add("all_equal_long", np.full(300_001, 0.1, np.float32))
    add("all_equal_3e4", np.full(100_000, np.float32(30000.002), np.float32))
    add("all_zero", np.zeros(4000, np.float32))
    add("constant_but_trimmed", _put(np.full(4000, 1.25, np.float32), [0, 3999], np.float32(9.0)))
    # tiny windows: 0, 1, 2 and 3 kept samples
    for k in (0, 1, 2, 3, 21, 22, 40):
        x = np.full(50, M4, np.float32)
        x[5:5 + k] = np.arange(k, dtype=np.float32) * np.float32(0.37) - np.float32(1.1)
        add("kept_%d" % k, x)
    # samples on bin edges: dyadic variances, integer magnitudes
    add("dyadic_two_levels", np.tile(np.array([0.0, 1.0], np.float32), 4000))
    add("dyadic_three_levels", np.tile(np.array([0.0, 0.5, 1.0, 0.5], np.float32), 3000))
    rng = np.random.default_rng(5)
    iq = rng.integers(-100, 101, (30_000, 2))
    mag = np.sqrt((iq.astype(np.float64) ** 2).sum(axis=1))
    add("int8_magnitudes_rounded", np.round(mag).astype(np.float32))
    lv = np.repeat(rng.integers(0, 2, 30_000 // 25 + 1), 25)[:30_000] * 60 + 20
    add("int_levels_small_noise", (lv + rng.integers(-1, 2, 30_000)).astype(np.float32))
    # rank windows and tiles
    for n in (TILE - 1, TILE, TILE + 1, 5 * TILE - 1, 5 * TILE + 1, 40 * TILE):
        add("n_%d" % n, _bimodal(n, n))
    x = _bimodal(30 * TILE, 7)
    for t in (3, 4, 10, 11, 12, 25):
        x[t * TILE:(t + 1) * TILE] = M4
    add("silent_tiles", x)
    x = np.full(20 * TILE, M4, np.float32)
    x[9 * TILE + 100:9 * TILE + 1900] = _bimodal(1800, 8)   # every kept sample in one tile
    add("window_in_one_tile", x)
    x = _bimodal(40 * TILE, 9)
    x[:TILE // 2] = M4   # 1024 dropped, so kept = 40*2048 - 1024 and the window starts mid-tile
    add("window_r0_mid_tile", x)
    x = np.full(40 * TILE, M4, np.float32)
    x[:20 * TILE] = _bimodal(20 * TILE, 10)   # kept = 20 tiles: r0 = 2048 = tile 1's first sample, r1 = 19 tiles
    add("window_on_tile_boundaries", x)
    add("max_size_mid_tile", _bimodal(30 * TILE, 11), 5 * TILE + 777)
    add("max_size_one", _bimodal(3 * TILE, 12), 1)
    add("max_size_two", _bimodal(3 * TILE, 13), 2)
    add("max_size_zero", _bimodal(3 * TILE, 14), 0)
    # far from zero relative to the spread
    for name, level, sigma in (("offset_1e3_near_2p20", 1000.0, 0.031), ("offset_5e3", 5000.0, 0.0316),
                               ("carrier_3e4_2e-3", 30000.0, 2e-3), ("carrier_3e4_0.5", 30000.0, 0.5),
                               ("carrier_ask_levels_3e4", None, None)):
        if level is None:
            x = _bimodal(60_000, 15, lo=30000.0, hi=30000.05, sigma=4e-3)
        else:
            x = (level + sigma * np.random.default_rng(16).standard_normal(60_000)).astype(np.float32)
        add(name, x)
    return out
