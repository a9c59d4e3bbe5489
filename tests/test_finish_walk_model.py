"""CPU: the pulse-table finish (finish.cu: stage B's per-tile firing count, stage C's first firing, stage D's warp walk in
k_finish_rows / fin_chunk), restated in numpy and checked row for row against the oracle's grab_pulse_lens.

The tile tables are built from the sample classes as the dense pass leaves them: per 2048-sample tile the head candidate (a run that
entered the tile reaches the tolerance inside it: head_rel), the staged candidates (runs that start in the tile and reach the
tolerance inside it: (position << 16) | (class + 1)), and stage B's class of the candidate before the tile.  The walk takes a tile's
staged words 32 at a time: the predecessor's class by a shift of one lane (lane 0: the carried class), the firings as a ballot
mask, each firing's row as the running row count plus the popcount of the lower lanes, and its previous firing as the highest
firing lane below it (positions grow with the lane), else the carried one."""
import numpy as np
import pytest

TILE = 2048
LANES = 32
FULL = (1 << LANES) - 1


def classes_to_qad(cls, mod):
    """a float32 qad array whose classes at center 0.0 are `cls` (-1: the modulation's noise sentinel)"""
    noise = np.float32(-4.0) if mod == "FSK" else np.float32(0.0)
    return np.where(cls < 0, noise, np.where(cls == 0, np.float32(-0.5), np.float32(0.5))).astype(np.float32)


def tile_tables(cls, tol):
    """head_rel, staged words and the class of the candidate preceding each tile (None: none before it)"""
    n = len(cls)
    ntiles = -(-n // TILE)
    edges = np.flatnonzero(np.diff(cls)) + 1
    starts = np.concatenate([[0], edges])
    ends = np.concatenate([edges, [n]])
    head_rel = [-1] * ntiles
    staged = [[] for _ in range(ntiles)]
    for s, e in zip(starts, ends):
        if e - s <= tol:
            continue
        p = s + tol
        t = p // TILE
        if s < t * TILE:
            head_rel[t] = p - t * TILE
        else:
            staged[t].append(((p - t * TILE) << 16) | (int(cls[s]) + 1))
    prev_cls = []
    last = None
    for t in range(ntiles):
        prev_cls.append(last)
        if staged[t]:
            last = (staged[t][-1] & 0xFFFF) - 1
        elif head_rel[t] >= 0:
            last = int(cls[t * TILE])
    return head_rel, staged, prev_cls


def walk_tile(t, cls, head_rel, staged, prev, pp, idx, rows=None, tol=0, is_ask=False, sps=1):
    """one tile's walk; returns (prev, pp, idx, fired, last_pos) and appends (row, state, length) to rows (stage D)"""
    base = t * TILE
    fired, last_pos = 0, -1

    def row(r, p, q, st):
        rec = p - q if q >= 0 else p + 1 - tol
        if is_ask and st == -1 and rec < sps:
            st = 0
        rows.append((r, st, rec))

    if head_rel[t] >= 0:
        c = int(cls[base])
        if c != prev:
            if rows is not None:
                row(idx, base + head_rel[t], pp, prev)
            fired += 1
            idx += 1
            last_pos = pp = base + head_rel[t]
        prev = c
    words = staged[t]
    for k in range(0, len(words), LANES):
        chunk = words[k:k + LANES]
        cnt = len(chunk)
        w = np.zeros(LANES, np.int64)
        w[:cnt] = chunk
        c = (w & 0xFFFF) - 1
        rel = w >> 16
        pc = np.concatenate([[prev], c[:-1]])                       # __shfl_up_sync(c, 1), lane 0: the carried class
        fire = (np.arange(LANES) < cnt) & (c != pc)
        fm = int(np.sum(fire.astype(np.int64) << np.arange(LANES)))  # __ballot_sync
        if rows is not None:
            for lane in np.flatnonzero(fire):
                lower = fm & ((1 << int(lane)) - 1)                     # firing lanes below this one
                r = idx + bin(lower).count("1")
                q = base + int(rel[lower.bit_length() - 1]) if lower else pp
                row(r, base + int(rel[lane]), q, int(pc[lane]))
        if fm:
            hl = fm.bit_length() - 1
            last_pos = pp = base + int(rel[hl])
        fired += bin(fm).count("1")
        idx += bin(fm).count("1")
        if cnt:
            prev = int(c[cnt - 1])
    return prev, pp, idx, fired, last_pos


def finish_model(cls, tol, is_ask, sps):
    """stages B..D as finish.cu runs them (one shard, no chain); ASK rows merged as ScanMergeRows merges them"""
    n = len(cls)
    cls_of_zero = 0   # 0.0 <= center 0.0
    prev0 = -1 if cls[0] < 0 else cls_of_zero
    head_rel, staged, prev_cls = tile_tables(cls, tol)
    ntiles = len(head_rel)
    # stage B's walk: each tile's firings after its first candidate; stage C adds the first one's against the preceding class
    row_off, prev_fired = [], []
    tot, lastp = 0, -1
    for t in range(ntiles):
        seq = ([(head_rel[t], int(cls[t * TILE]))] if head_rel[t] >= 0 else []) + [(w >> 16, (w & 0xFFFF) - 1) for w in staged[t]]
        fired, last_rel = 0, -1
        for (_, c0), (p1, c1) in zip(seq, seq[1:]):
            if c1 != c0:
                fired, last_rel = fired + 1, p1
        prev = prev_cls[t] if prev_cls[t] is not None else prev0
        if seq and seq[0][1] != prev:
            fired += 1
            if last_rel < 0:
                last_rel = seq[0][0]
        row_off.append(tot)
        prev_fired.append(lastp)
        tot += fired
        if last_rel >= 0:
            lastp = t * TILE + last_rel
    # stage D: every tile's rows land at its row offset
    rows = []
    for t in range(ntiles):
        prev = prev_cls[t] if prev_cls[t] is not None else prev0
        prev, pp, idx, _, _ = walk_tile(t, cls, head_rel, staged, prev, prev_fired[t], row_off[t], rows, tol, is_ask, sps)
    fired = idx
    out = np.zeros((fired + 1, 2), np.int64)
    for r, st, rec in rows:
        out[r] = (st, rec)
    k = fired
    if is_ask or fired < n:
        out[fired] = (prev, n - 1 - pp if pp >= 0 else n - tol)
        k += 1
    out = out[:k]
    if not is_ask or k == 0:
        return out
    merged = []
    has_tail = k > fired
    for r in range(k):
        if has_tail and r == k - 1 and len(merged) >= n:
            break
        if merged and merged[-1][0] == out[r, 0]:
            merged[-1][1] += int(out[r, 1])
        else:
            merged.append([int(out[r, 0]), int(out[r, 1])])
    return np.array(merged, np.int64).reshape(-1, 2)


def random_classes(n, seed, short=3, long=0, p_long=0.0, noise=0.2):
    """runs of 1..short samples, with probability p_long a run of up to `long`; each run's class differs from the previous one"""
    rng = np.random.default_rng(seed)
    out, c, total = [], int(rng.integers(-1, 2)), 0
    while total < n:
        L = int(rng.integers(1, long + 1)) if long and rng.random() < p_long else int(rng.integers(1, short + 1))
        out.append(np.full(L, c, np.int64))
        total += L
        choices = [x for x in (-1, 0, 1) if x != c]
        c = choices[0] if rng.random() < 0.5 else choices[1]
        if c == -1 and rng.random() > noise:
            c = choices[1] if choices[0] == -1 else choices[0]
    return np.concatenate(out)[:n]


def check(oracle, cls, tol, mod="FSK", sps=100):
    rows = finish_model(cls, tol, mod == "ASK", sps)
    ref = oracle.grab_pulse_lens(classes_to_qad(cls, mod), 0.0, tol, mod, sps)
    assert np.array_equal(rows, ref), (tol, mod, rows[:8], ref[:8])
    return rows


@pytest.mark.parametrize("mod", ["FSK", "ASK"])
@pytest.mark.parametrize("tol", [0, 1, 5, 31, 32, 33, 3000])
def test_random_classes(oracle, tol, mod):
    for seed in range(3):
        cls = random_classes(5 * TILE + 777, seed=seed + 10 * tol, short=max(3, tol + 3), long=6000, p_long=0.02)
        check(oracle, cls, tol, mod, sps=max(4, tol))


def test_tolerance_zero_fills_the_staging_row(oracle):
    """a class change on almost every sample: ~1000 staged candidates per tile, more than 32 chunks of the walk"""
    _, staged, _ = tile_tables(random_classes(3 * TILE, seed=1, short=2), 0)
    assert max(len(s) for s in staged) > 900
    for mod in ("FSK", "ASK"):
        check(oracle, random_classes(3 * TILE + 5, seed=1, short=2), 0, mod)


def test_head_candidates_with_and_without_staged(oracle):
    cls = np.zeros(4 * TILE, np.int64)
    cls[TILE - 3:2 * TILE + 10] = 1      # enters tile 1 and reaches tolerance 5 there: head candidate, no staged one
    cls[3 * TILE - 2:3 * TILE + 50] = -1  # head candidate of tile 3 ...
    cls[3 * TILE + 50:3 * TILE + 60] = 1  # ... followed by staged ones
    head_rel, staged, _ = tile_tables(cls, 5)
    assert head_rel[1] >= 0 and head_rel[3] >= 0 and staged[3] and not staged[1]
    check(oracle, cls, 5)


def test_tiles_without_candidates_and_long_tolerance(oracle):
    cls = np.zeros(10 * TILE + 3, np.int64)
    cls[7000:23000] = 1
    cls[23000:23003] = -1
    cls[23003:41000] = 1
    for tol in (0, 5, 2047, 2048, 5000, 20000):
        check(oracle, cls, tol)
        check(oracle, cls, tol, "ASK")


def test_first_firing_of_the_capture(oracle):
    for first in (-1, 0, 1):
        cls = np.full(3 * TILE, first, np.int64)
        cls[100:] = 1 - abs(first)
        check(oracle, cls, 5)


def test_ask_short_pauses_merge(oracle):
    cls = np.ones(6 * TILE, np.int64)
    cls[1000:1030] = -1                  # pause shorter than a symbol: relabelled 0 ...
    cls[1030:1060] = 0                   # ... and merged with the zero after it
    cls[5000:5500] = -1                  # a long pause stays -1
    rows = check(oracle, cls, 5, "ASK", sps=100)
    assert (rows[:, 0] == 0).any() and (rows[:, 0] == -1).any()


def test_tail_row_rule(oracle):
    """every sample fires at tolerance 0 when the classes alternate from the first sample on: n firings, no tail row"""
    n = 2 * TILE + 17
    cls = (np.arange(n) + 1) % 2
    rows = check(oracle, cls, 0)
    assert len(rows) == n
    cls2 = cls.copy()
    cls2[0] = 0                          # samples 0 and 1 form one run: n - 2 firings and the tail row
    assert len(check(oracle, cls2, 0)) == n - 1
