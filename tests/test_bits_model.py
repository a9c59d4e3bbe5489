"""CPU check of the array restatement behind bits.cu: the same maps / prefix sums in numpy == the sequential
_ppseq_to_bits port (which test_gpu_objects pins against the reference's golden bit strings)."""
import numpy as np

from urh_b200.signalprocessing.ProtocolAnalyzer import ProtocolAnalyzer as PA


def _oracle_ppseq_to_bits(*a, **k):
    """the sequential CPU restatement of ProtocolAnalyzer._ppseq_to_bits lives in the test oracle, not in the product"""
    from oracle import oracle
    return oracle.ppseq_to_bits(*a, **k)



def model(rows, sps, bps, pt):
    """the restatement in flat arrays, as urh_fetch_bits returns them: (bits uint8[B], msg_off int64[M+1], pauses int64[M],
    pos int64[P]); message m is bits[msg_off[m]:msg_off[m+1]] with positions pos[msg_off[m] + 2m : msg_off[m+1] + 2m + 2]
    (one fewer for a last message that no pause row closes).  Loop-free, so it serves tables of millions of rows."""
    rows = np.asarray(rows, np.int64).reshape(-1, 2)
    k = len(rows)
    if k == 0:
        return np.zeros(0, np.uint8), np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64)
    kind, ns = rows[:, 0], rows[:, 1]
    first = 1 if kind[0] == -1 else 0
    f = ns / float(sps)
    nsym = f.astype(np.int64)
    nsym += (f - nsym > 0.5)
    idx = np.arange(k)
    live = idx >= first
    is_pause = kind == -1
    zero = live & is_pause & ((nsym <= pt) | (pt == 0))
    long_ = live & is_pause & ~zero
    data = live & ~is_pause
    nbits = np.where(zero | data, nsym * bps, 0)
    has = data & (nsym > 0)
    total = np.concatenate([[0], np.cumsum(ns)])
    seg = np.concatenate([[0], np.cumsum(long_)])[:k]
    nseg = int(long_.sum()) + 1
    seg_has = np.zeros(nseg + 1, np.int64)
    seg_has[seg[has]] = 1
    seg_msg = np.concatenate([[0], np.cumsum(seg_has)])
    eff = np.where(seg_has[seg] == 1, nbits, 0)
    bitoff = np.concatenate([[0], np.cumsum(eff)])
    M, B = int(seg_has[:nseg].sum()), int(bitoff[-1])
    final_open = bool(seg_has[nseg - 1])
    msg_off = np.zeros(M + 1, np.int64)
    pauses = np.zeros(M, np.int64)
    pos = np.zeros(B + 2 * M, np.int64)
    # a long pause closes its segment's message
    i = np.nonzero(long_ & (seg_has[seg] == 1))[0]
    m = seg_msg[seg[i]]
    msg_off[m + 1] = bitoff[i]
    pauses[m] = ns[i]
    pos[bitoff[i] + 2 * m] = total[i]
    pos[bitoff[i] + 2 * m + 1] = total[i] + ns[i]
    if final_open:
        msg_off[M] = B
        pauses[M - 1] = ns[-1] if kind[-1] == -1 else 0
        pos[B + 2 * (M - 1)] = total[k]
    # every bit: its row, its index inside the row, the row's symbol digits MSB first
    r = np.repeat(idx, eff)
    b = np.arange(B, dtype=np.int64) - bitoff[r]
    bits = np.where(data[r], (kind[r] >> (bps - 1 - b % bps)) & 1, 0).astype(np.uint8)
    spb = int(sps / bps)
    pos[np.arange(B, dtype=np.int64) + 2 * seg_msg[seg[r]]] = total[r] + b * spb
    P = B + 2 * M - (1 if final_open else 0)
    return bits, msg_off, pauses, pos[:P]


def as_messages(flat):
    """model()'s flat arrays -> per-message lists, the shape the sequential port returns"""
    bits, msg_off, pauses, pos = flat
    M = len(pauses)
    out_bits = [bits[msg_off[m]:msg_off[m + 1]].tolist() for m in range(M)]
    out_pos = [pos[msg_off[m] + 2 * m: min(msg_off[m + 1] + 2 * m + 2, len(pos))].tolist() for m in range(M)]
    return out_bits, pauses.tolist(), out_pos


def test_model_equals_sequential_port():
    rng = np.random.default_rng(7)
    for trial in range(400):
        bps = int(rng.choice([1, 2, 3]))
        pt = int(rng.choice([8, 0, 1, 3]))
        sps = int(rng.choice([1, 2, 7, 10, 100]))
        k = int(rng.integers(1, 60))
        kinds = rng.integers(-1, 1 << bps, k)
        ns = np.where(rng.random(k) < 0.15, rng.integers(9, 30, k) * sps, rng.integers(0, 5 * sps + 1, k))
        rows = np.stack([kinds, ns], axis=1).astype(np.int64)
        hb, hp, hpos = _oracle_ppseq_to_bits(rows, sps, bps, pause_threshold=pt)
        mb, mp, mpos = as_messages(model(rows, sps, bps, pt))
        assert [list(x) for x in hb] == mb, (trial, rows.tolist())
        assert list(hp) == mp, (trial, rows.tolist())
        assert [list(x) for x in hpos] == mpos, (trial, rows.tolist())
