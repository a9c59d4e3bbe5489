"""Float32 qad arrays with digitizer parameters at the edges of grab_pulse_lens (signal_functions.pyx:392-495), each with a name.

tests/test_oracle.py pins the oracle's grab_pulse_lens to the reference's on them (recorded in tests/golden/ref_pulse_edges.json);
tests/test_gpu_pulse_edges.py runs them through every device digitizer entry point against the oracle.  They cover:
* orders 1 .. 256 (bits per symbol 0, 1, 2, 3, 4, 8) with thresholds at spacing 0.1, 0 (coinciding), -0.3 (descending: "the first
  k with s <= thr[k]" is no longer "the number of thresholds below s"), NaN, 1e-45 and 1e38 (infinite thresholds), around centers
  0, -4, NaN, +-inf and one just below and one just above 0 (the initial state classifies the literal 0.0, not samples[0]);
* samples on each threshold and one float either side of it, +-0 (0 is the ASK and unknown sentinel, -0.0 the QAM one: 0.0f * -4.0f),
  -4 and pred(-4), a value below -4, NaN (class order - 1) and +-inf, at even and odd positions and on tile (2048-sample) edges;
* every modulation string: ASK, FSK, PSK, OQPSK, QAM and an unknown one (sentinel 0);
* run geometry: class changes at 2047 / 2048 / 2049, runs of tol and tol + 1 ending on a tile edge, whole-tile runs, an all-noise
  tile and one with a single noise sample, tiles full of candidates (tolerance 0 and 1, alternating);
* tolerances 0, 1, 31, 32, 33, 2047, 2048, 2049 and 65535, and tolerance >= n (the only row has a negative length);
* the ASK relabel of short pauses (pulse - tolerance < samples_per_symbol) at sps - 1, sps and sps + 1, with sps 0, 1 and 2^32 - 1;
* the tail row dropped when the table already holds n rows: FSK, ASK without merges and ASK whose merges bring the count back under
  n, at n = 2047, 2048, 2049, 4097 and 2^20 + 1."""
import numpy as np

TILE = 2048
F = np.float32
NAN, INF = F(np.nan), F(np.inf)
M4 = F(-4.0)
MODS = ["ASK", "FSK", "PSK", "OQPSK", "QAM", "OOK"]   # OOK: not a modulation grab_pulse_lens knows, sentinel 0
SPACINGS = [0.1, 0.0, -0.3, float("nan"), 1e-45, 1e38]
CENTERS = [0.0, -4.0, float("nan"), float("inf"), float("-inf"), -0.25, 0.25]
SPS_MAX = 2 ** 32 - 1


def pred(x):
    return np.nextafter(F(x), F(-np.inf))


def succ(x):
    return np.nextafter(F(x), F(np.inf))


def thresholds(center, spacing, order):
    """get_center_thresholds (signal_functions.pyx:380-390) in float32"""
    n = order // 2
    c, sp = F(center), F(spacing)
    with np.errstate(over="ignore", invalid="ignore"):   # spacing 1e38 and infinite centers
        lo = [c - F(n - (i + 1)) * sp for i in range(n)]
        hi = [c + F(i + 1 - n) * sp for i in range(n, order - 1)]
    return np.array(lo + hi, dtype=F)


def _unique_words(v):
    v = np.asarray(v, dtype=F)
    _, idx = np.unique(v.view(np.uint32), return_index=True)
    return v[np.sort(idx)]


def _values(thr):
    """every sample value a classifier can get wrong for these thresholds"""
    v = [F(0.0), F(-0.0), M4, pred(M4), succ(M4), F(-4.5), NAN, INF, -INF, F(1e38), F(-1e38), F(1e-45), F(-1e-45)]
    for t in thr:
        v += [pred(t), t, succ(t)]
    return _unique_words(v)


def _values_array(thr, seed):
    """the values in runs of 1, 1, 2 and 3 samples, shuffled, over a little more than two tiles; special values on the first and
    last sample of each tile and on the last sample"""
    rng = np.random.default_rng(seed)
    vals = _values(thr)
    n = 2 * TILE + 3
    parts, total = [], 0
    while total < n:
        order = rng.permutation(len(vals))
        reps = np.array([1, 1, 2, 3])[np.arange(len(vals)) % 4]
        parts.append(np.repeat(vals[order], reps))
        total += len(parts[-1])
    x = np.concatenate(parts)[:n].astype(F)
    edge = [F(-0.0), M4, NAN, F(0.0), pred(M4), INF]
    for j, p in enumerate((TILE - 1, TILE, 2 * TILE - 1, 2 * TILE, n - 1)):
        x[p] = edge[(j + seed) % len(edge)]
    return x


class Case:
    __slots__ = ("name", "x", "center", "tol", "mod", "sps", "bps", "spacing")

    def __init__(self, name, x, center, tol, mod, sps, bps, spacing):
        self.name, self.x = name, np.ascontiguousarray(x, dtype=F)
        self.center, self.tol, self.mod, self.sps, self.bps, self.spacing = float(center), int(tol), mod, int(sps), int(bps), float(spacing)

    def args(self):
        """grab_pulse_lens(x, *args)"""
        return self.center, self.tol, self.mod, self.sps, self.bps, self.spacing


def _levels(n, seed, lo=-1.0, hi=1.0, run=(1, 60)):
    rng = np.random.default_rng(seed)
    r = rng.integers(run[0], run[1], n // run[0] + 1)
    return np.repeat(np.where(np.arange(len(r)) % 2 == 0, hi, lo), r)[:n].astype(F)


def _alternating(n, first, second):
    x = np.empty(n, F)
    x[0::2] = first
    x[1::2] = second
    return x


def cases():
    """every Case, names unique"""
    out = []

    def add(*a):
        out.append(Case(*a))

    # ---- orders, threshold layouts and sample values ---------------------------------------------------------------------------------
    i = 0
    for bps in (0, 1, 2, 3, 4, 8):
        layouts = [(0.0, 0.1), (0.25, -0.3)] if bps == 0 else [(c, sp) for sp in SPACINGS for c in CENTERS]
        for c, sp in layouts:
            thr = thresholds(c, sp, 1 << bps)
            x = _values_array(thr, seed=1000 * bps + i)
            mod = MODS[i % len(MODS)]
            tol = (0, 1, 2)[(i // len(MODS)) % 3]
            sps = (0, 1, 7, SPS_MAX)[(i // 3) % 4]
            add("values_bps%d_c%s_sp%s_%s" % (bps, c, sp, mod), x, c, tol, mod, sps, bps, sp)
            i += 1
    # every modulation string on one array holding +-0, -4 and its neighbours, NaN and +-inf
    x = _values_array(thresholds(0.0, 0.1, 4), seed=7)
    for mod in MODS:
        for tol in (0, 3):
            add("mods_%s_tol%d" % (mod, tol), x, 0.0, tol, mod, 5, 2, 0.1)
    # QAM: -0.0 and 0.0 are both the sentinel; ASK / unknown: both are 0 too; FSK: neither is
    x = np.tile(np.array([0.5, -0.0, -0.0, 0.7, 0.0, 0.0, 0.0, -0.5, -0.0, 0.3], F), 420)
    for mod in ("QAM", "ASK", "FSK", "OOK"):
        add("signed_zero_%s" % mod, x, 0.1, 1, mod, 3, 1, 0.1)

    # ---- run geometry -------------------------------------------------------------------------------------------------------------
    n = 3 * TILE + 5
    for k in (TILE - 1, TILE, TILE + 1):
        x = np.full(n, F(0.8), F)
        x[k:] = F(-0.8)
        x[k + 700: k + 703] = M4
        for tol in (0, 1, 5):
            add("change_at_%d_tol%d" % (k, tol), x, 0.0, tol, "FSK", 10, 1, 0.1)
    for tol in (0, 1, 31, 32, 33):
        for length in (tol, tol + 1):
            if length == 0:
                continue
            x = _levels(5 * TILE + 17, seed=tol, run=(tol + 2, tol + 40)) if tol else _levels(5 * TILE + 17, seed=1, run=(2, 9))
            for end in (TILE, 2 * TILE, 4 * TILE):   # a run of `length` samples ending on the tile's last sample
                x[end - length - 1] = F(-1.0)
                x[end - length: end] = F(1.0)
                x[end] = F(-1.0)
            x[3 * TILE: 3 * TILE + length] = F(1.0)  # and one starting on a tile's first sample
            x[3 * TILE + length] = F(-1.0)
            for mod in ("FSK", "ASK"):
                add("run_%d_tol%d_%s" % (length, tol, mod), x, 0.0, tol, mod, 4, 1, 0.1)
    x = _levels(6 * TILE + 100, seed=3)
    x[TILE: 2 * TILE] = F(1.0)            # a whole tile of one class
    x[2 * TILE: 3 * TILE] = F(-1.0)       # and the next of the other
    x[3 * TILE: 4 * TILE] = M4            # an all-noise tile
    x[4 * TILE + 1000] = M4               # a single noise sample
    x[5 * TILE: 6 * TILE] = F(1.0)
    x[5 * TILE + 2047] = M4               # a noise sample on a tile's last position
    for tol in (0, 1, 31):
        add("whole_tiles_tol%d" % tol, x, 0.0, tol, "FSK", 10, 1, 0.1)
    xa = np.where(x == M4, F(0.0), x)     # the same for ASK (sentinel 0)
    add("whole_tiles_ask", xa, 0.0, 2, "ASK", 10, 1, 0.1)
    # candidates filling a tile: every sample (tolerance 0), every second sample (tolerance 1)
    x = _alternating(3 * TILE + 1, F(1.0), F(-1.0))
    add("alternating_tol0", x, 0.0, 0, "FSK", 1, 1, 0.1)
    add("alternating_tol0_bps2", np.tile(np.array([-1, -0.1, 0.1, 1], F), TILE), 0.0, 0, "FSK", 1, 2, 0.2)
    add("pairs_tol1", np.repeat(_alternating(3 * TILE // 2 + 1, F(1.0), F(-1.0)), 2), 0.0, 1, "FSK", 1, 1, 0.1)
    add("alternating_noise_tol0", _alternating(2 * TILE + 3, F(1.0), M4), 0.0, 0, "FSK", 1, 1, 0.1)

    # ---- tolerances ---------------------------------------------------------------------------------------------------------------
    for tol in (0, 1, 31, 32, 33, 2047, 2048, 2049, 65535):
        rng = np.random.default_rng(tol + 5)
        runs = np.maximum(1, tol + rng.integers(-2, 3, 40))
        runs[::7] = 1
        lv = np.repeat(rng.integers(0, 3, len(runs)), runs)
        x = np.array([-1.0, 1.0, -4.0], F)[lv]
        for mod in ("FSK", "ASK"):
            add("tol_%d_%s" % (tol, mod), x if mod == "FSK" else np.where(x == M4, F(0.0), x), 0.0, tol, mod, 3, 1, 0.1)
    for n in (1, 2, 5):
        for tol in (n - 1, n, n + 1, 65535):
            for mod, first in (("FSK", F(1.0)), ("FSK", M4), ("ASK", F(0.0))):
                x = np.full(n, first, F)
                add("tol_ge_n_%d_tol%d_%s_%s" % (n, tol, mod, "noise" if first in (M4, 0.0) else "data"), x, 0.0, tol, mod, 2, 1, 0.1)

    # ---- the ASK relabel of short pauses ------------------------------------------------------------------------------------------
    for sps in (0, 1, 10, SPS_MAX):
        parts = []
        for pause in ((9, 10, 11) if sps == 10 else (1, 2, 3, 7)):
            parts += [np.full(30, F(0.9)), np.full(pause, F(0.0)), np.full(25, F(0.2)), np.full(pause + 2, F(0.0))]
        x = np.tile(np.concatenate(parts), 40)
        for tol in (0, 2):
            add("ask_relabel_sps%d_tol%d" % (sps, tol), x, 0.5, tol, "ASK", sps, 1, 0.1)

    # ---- the tail row dropped at n rows -----------------------------------------------------------------------------------------
    for n in (2047, 2048, 2049, 4097, 2 ** 20 + 1):
        # class of 0.0 is 0, samples[0] is class 1, every sample changes class: n firings
        add("tail_drop_fsk_%d" % n, _alternating(n, F(1.0), F(-1.0)), 0.0, 0, "FSK", 1, 1, 0.1)
        add("tail_drop_ask_%d" % n, _alternating(n, F(0.9), F(0.2)), 0.5, 0, "ASK", 1, 1, 0.1)
        # pauses of one sample relabelled to 0 merge with their neighbours: n firings, fewer rows, the tail row stays
        x = np.resize(np.array([0.9, 0.0, 0.2, 0.0], F), n)
        add("tail_merge_ask_%d" % n, x, 0.5, 0, "ASK", 5, 1, 0.1)
        # one pause sample between two 0.2 samples: still n firings, two merges, so the tail row is appended to n - 2 rows
        x = _alternating(n, F(0.9), F(0.2))
        x[n // 2 - (n // 2) % 2] = F(0.0)
        add("tail_merge_one_ask_%d" % n, x, 0.5, 0, "ASK", 5, 1, 0.1)
    add("tail_drop_bps2_4097", np.resize(np.array([1.0, -1.0, 0.15, -0.15], F), 4097), 0.0, 0, "FSK", 1, 2, 0.1)

    names = [c.name for c in out]
    assert len(names) == len(set(names)), "case names must be unique"
    return out
