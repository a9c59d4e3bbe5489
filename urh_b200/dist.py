"""One capture sharded by contiguous sample range over the GPUs of one box (SURVEY §8e).

One process per GPU (launched by torchrun).  ``torch.distributed`` (gloo) is the launcher plumbing: rendezvous and
the exchange of tiny host-side descriptors; the data path between GPUs is NCCL over NVLink, driven from
liburh_b200 (nccl.cu): the 1-sample halo, the all-reduce of the global noise statistics and the digitizer's three
small all-gathers.  Per rank the sample-rate work is exactly the single-GPU dense pass.

Protocol of the sharded digitizer, one library call per rank (exactness argument in DESIGN.md §6):
  1. every rank: dense pass over its shard (+1 halo sample for the FSK conjugate product) -> tile table;
  2. the tile-level finish (finish.cu) on every rank, with three NCCL all-gathers of 32, 16 and 16 bytes per rank on the
     context stream, each folded over the ranks before it: the run that ends right before the shard, the class of the
     candidate preceding it and the position of the last firing before it;
  3. every rank ends with the (state, length) rows of its own shard; ``merge_shard_rows`` joins them, merging equal states
     that meet at a shard edge.
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from .device import DeviceArray, to_device


# ---- pure host logic (unit-tested on CPU with gloo, tests/test_dist_cpu.py) -----------------------------------------
def fold_carry(summaries):
    """summaries: list of (last_cls, last_len, whole) per rank, in rank order.
    Returns for every rank the run that ends right before its shard: None for rank 0, else (cls, len)."""
    out = []
    carry = None  # (cls, len, whole)
    for cls, length, whole in summaries:
        out.append(None if carry is None else (carry[0], carry[1]))
        if carry is not None and whole and cls == carry[0]:
            carry = (cls, carry[1] + length, carry[2])
        else:
            carry = (cls, length, bool(whole) and carry is None)
    return out


def shard_bounds(n_total: int, world: int, align: int = 2048):
    """contiguous shards whose boundaries are multiples of `align` (the dense pass's tile), last one takes the rest"""
    per = (n_total // world) // align * align
    if per == 0:
        per = n_total
    bounds = []
    start = 0
    for r in range(world):
        end = n_total if r == world - 1 else min(n_total, start + per)
        bounds.append((start, end))
        start = end
    return bounds


def combine_noise_chunks(n_total, chunksize, nchunks, partial_sums, partial_maxs):
    """Global end-aligned noise chunks (AutoInterpretation.py:66-72) from per-rank partial (sum, max) arrays that were
    all-reduced element-wise (sum / max) — identity here; kept for symmetry with the CPU test."""
    return np.asarray(partial_sums, dtype=np.float64), np.asarray(partial_maxs, dtype=np.float64)


class HostExchange(object):
    """tiny host-side collectives over torch.distributed (gloo)"""

    def __init__(self):
        import torch.distributed as dist

        self.dist = dist
        self.rank = dist.get_rank()
        self.world = dist.get_world_size()

    def allgather(self, obj):
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    def broadcast(self, obj, src=0):
        box = [obj]
        self.dist.broadcast_object_list(box, src=src)
        return box[0]

    def barrier(self):
        self.dist.barrier()


def init_nccl(ctx: _lib.Context, hx: HostExchange):
    """create the NCCL communicator of liburh_b200 for this context (id from rank 0 via the host exchange)"""
    buf = C.create_string_buffer(128)
    if hx.rank == 0:
        rc = ctx.lib.urh_nccl_unique_id(buf)
        if rc != 0:
            raise RuntimeError("urh_nccl_unique_id failed (libnccl.so.2 not loadable?)")
    ident = hx.broadcast(bytes(buf.raw) if hx.rank == 0 else None, src=0)
    ctx.check(ctx.lib.urh_nccl_init(ctx.handle, C.c_char_p(ident), hx.rank, hx.world))


class ShardBuffer(object):
    """Device buffer [pad][halo][shard samples...][right]: the shard starts 256-byte aligned (full-line warp loads), the halo
    samples sit right before it, the optional right halo (the next shard's first samples) right after it."""

    def __init__(self, ctx, n_local, dtype=np.float32, halo=1, right=0):
        self.ctx = ctx
        self.n = int(n_local)
        self.dtype = np.dtype(dtype)
        self.halo_len = int(halo)
        self.right_len = int(right)
        unit = 256 // (2 * self.dtype.itemsize)  # samples per 256 bytes
        self.pad = ((self.halo_len + unit - 1) // unit) * unit  # samples before the shard (keeps 256 B alignment)
        self.buf = DeviceArray(ctx, (self.n + self.pad + self.right_len, 2), self.dtype)
        self.shard = self.buf[self.pad: self.pad + self.n]
        self.halo = self.buf[self.pad - self.halo_len: self.pad]
        self.right = self.buf[self.pad + self.n: self.pad + self.n + self.right_len]

    def window(self, left, right):
        """the shard with `left` samples before it and `right` after it: [g0 - left, g1 + right) of the capture"""
        assert 0 <= left <= self.halo_len and 0 <= right <= self.right_len
        return self.buf[self.pad - left: self.pad + self.n + right]


def exchange_halo(ctx, hx, sb: ShardBuffer):
    """rank r receives the last `halo_len` samples of rank r-1's shard (NCCL all-gather of the tails).  Every rank checks every
    shard that supplies a halo against it before the NCCL collective, so a short shard raises ValueError on every rank alike."""
    h = sb.halo_len
    shapes = hx.allgather((sb.n, h))
    if any(hq != h for _, hq in shapes):
        raise ValueError("exchange_halo: the ranks hold halos of %s samples; they must be equal" % sorted(set(hq for _, hq in shapes)))
    for q, (nq, _) in enumerate(shapes[:-1]):
        if nq < h:
            raise ValueError("exchange_halo: shard %d (%d samples) is shorter than the %d-sample halo shard %d needs" % (q, nq, h, q + 1))
    tail = sb.buf[sb.pad + sb.n - h: sb.pad + sb.n]   # the last rank's tail is sent but not used: it may reach into its halo
    allv = DeviceArray(ctx, (hx.world * h, 2), sb.dtype)
    ctx.check(ctx.lib.urh_nccl_allgather(ctx.handle, C.c_void_p(tail.ptr), C.c_void_p(allv.ptr), tail.nbytes))
    if hx.rank > 0:
        src = allv[(hx.rank - 1) * h: hx.rank * h]
        ctx.check(ctx.lib.urh_memcpy_d2d(ctx.handle, C.c_void_p(sb.halo.ptr), C.c_void_p(src.ptr), src.nbytes))
    ctx.sync()


def costas_halo(ctx) -> int:
    return int(ctx.lib.urh_costas_halo_samples())


def resolve_psk_chain(hyps):
    """Pure host logic of the sharded Costas loop (unit-tested on the CPU).  ``hyps[r]`` = list of (start_state, end_state) per
    hypothesis of rank r, states as raw 8-byte keys; rank 0 has one entry (its true run).  Returns (picks, first_unresolved):
    picks[r] = hypothesis of rank r whose start state equals the true end state of rank r-1, for r < first_unresolved;
    first_unresolved = world when every shard is resolved."""
    picks = [0]
    state = hyps[0][0][1]
    for r in range(1, len(hyps)):
        match = [h for h, (start, _) in enumerate(hyps[r]) if start == state]
        if not match:
            return picks, r
        picks.append(match[0])
        state = hyps[r][match[0]][1]
    return picks, len(hyps)


def afp_demod_psk_sharded(ctx, rank, world, sb: ShardBuffer, noise_mag, mod_order, costas_loop_bandwidth, d_out):
    """PSK demodulation (Costas loop) of a capture sharded over the ranks, bit-identical to the serial loop (the run between the
    library calls lives on ``ctx``).  Every rank
    speculates over its shard concurrently (the expensive pass) AND hops over it under each hypothesis "my shard starts in
    candidate h's start state" — what a locked loop of the preceding shard ends in, bit for bit.  One all-gather of
    (start, end) state pairs lets every rank pick its hypothesis (``resolve_psk_chain``); nothing waits for a neighbour.
    Only a shard whose predecessor ends in no hypothesis' start state (it begins inside a gap that carries a frozen or creeping
    loop state) falls back to the rank-to-rank hand-over from that shard on.  sb needs a halo of costas_halo() samples."""
    lib = ctx.lib
    if world > 1 and sb.halo_len < costas_halo(ctx):   # checked on rank 0 too, so every rank raises alike
        raise ValueError("afp_demod_psk_sharded: the shard buffer's halo (%d samples) is shorter than the Costas warm-up (%d)"
                         % (sb.halo_len, costas_halo(ctx)))
    ctx.check(lib.urh_costas_shard_speculate(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, int(rank == 0),
                                             float(noise_mag), int(mod_order), float(costas_loop_bandwidth), C.c_void_p(d_out.ptr)))
    mine = np.zeros((4, 4), dtype=np.float32)
    count = C.c_int(0)
    ctx.check(lib.urh_costas_shard_hypotheses(ctx.handle, mine.ctypes.data_as(C.c_void_p), C.byref(count)))
    mine[count.value:] = np.nan
    payload = np.concatenate([mine.reshape(-1).view(np.int32).astype(np.int64), [count.value]]).astype(np.int64)
    every = nccl_allgather_wide(ctx, world, payload)
    hyps = []
    for r in range(world):
        cnt = int(every[r, -1])
        raw = every[r, :16].astype(np.int32).view(np.float32).reshape(4, 4)
        hyps.append([(raw[h, 0:2].tobytes(), raw[h, 2:4].tobytes()) for h in range(cnt)])
    picks, unresolved = resolve_psk_chain(hyps)
    state = np.zeros(2, dtype=np.float32)
    if rank < unresolved:
        ctx.check(lib.urh_costas_shard_adopt(ctx.handle, picks[rank], state.ctypes.data_as(C.c_void_p)))
    if unresolved < world:
        # hand-over from the first unresolved shard on: its predecessor's end state is known exactly
        carry = np.frombuffer(hyps[unresolved - 1][picks[unresolved - 1]][1], dtype=np.float32).copy()
        for turn in range(unresolved, world):
            out = np.zeros(2, dtype=np.float32)
            if turn == rank:
                ctx.check(lib.urh_costas_shard_resolve(ctx.handle, carry.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
                state = out
            allv = np.empty((world, 2), dtype=np.float32)
            ctx.check(lib.urh_nccl_allgather_host(ctx.handle, out.ctypes.data_as(C.c_void_p), allv.ctypes.data_as(C.c_void_p), out.nbytes))
            carry = allv[turn].copy()
    return state


def nccl_allgather_wide(ctx, world, values):
    """all-gather an int64 vector per rank over NCCL (pinned staging) -> array [world, len(values)]"""
    send = np.ascontiguousarray(values, dtype=np.int64)
    recv = np.empty((world, len(send)), dtype=np.int64)
    ctx.check(ctx.lib.urh_nccl_allgather_host(ctx.handle, send.ctypes.data_as(C.c_void_p), recv.ctypes.data_as(C.c_void_p), send.nbytes))
    return recv


def demod_digitize_distributed(ctx, rank, world, sb: ShardBuffer, global_offset, n_total, noise_mag, mod_type, center, tolerance,
                               samples_per_symbol, bits_per_symbol=1, center_spacing=0.1, d_qad=None, fetch=True, qad_source=None):
    """Sharded FSK/ASK demod + digitize with a DISTRIBUTED finish: no gather, every rank ends with the rows of its own
    shard (``merge_shard_rows`` joins them).  One library call per rank (urh_shard_digitize): the dense pass, then the
    tile-level finish whose three 16-byte exchanges (run carry / class of the last candidate / position of the last firing)
    are NCCL all-gathers enqueued on the context stream — the host waits once, for the row count.
    ``qad_source``: the shard is already demodulated (float32 DeviceArray) -> digitize from it instead of the IQ samples."""
    lib = ctx.lib
    code = _lib.demod_mod_code(mod_type)
    k = C.c_int64(0)
    ctx.check(lib.urh_shard_digitize(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype),
                                     C.c_void_p(qad_source.ptr if qad_source is not None else 0), sb.n, int(rank > 0), float(noise_mag), code,
                                     float(center), int(tolerance), int(samples_per_symbol), int(bits_per_symbol), float(center_spacing),
                                     C.c_void_p(d_qad.ptr if d_qad is not None else 0), int(global_offset), int(n_total), C.byref(k)))
    if not fetch:
        return int(k.value)
    rows = np.empty((k.value, 2), dtype=np.int64)
    if k.value:
        ctx.check(lib.urh_fetch_pulses(ctx.handle, rows.ctypes.data_as(C.c_void_p), k.value))
    return rows


def center_protocol(rank, world, kept, window_stats, histogram, allgather_i64, allreduce_sum_i64, max_size=None):
    """The exchange behind a capture-wide detect_center, independent of where the numbers come from (GPU + NCCL in
    ``detect_center_distributed``; numpy + gloo in tests/test_dist_cpu.py).
      kept                      number of samples this shard keeps (qad > -4)
      window_stats(lr0, lr1)    -> [count, min, max, sum, sumsq] of the kept samples of LOCAL rank [lr0, lr1)
      histogram(lr0, lr1, edges)-> int64 counts of those samples for np.histogram(…, bins=edges)
      allgather_i64(values)     -> array [world, len(values)]; allreduce_sum_i64(array) -> array
    Every rank returns the same center (or None)."""
    from .ainterpretation.AutoInterpretation import center_rank_window, center_stats_from_window, pick_center_from_histogram, \
        center_bin_edges
    counts = np.asarray(allgather_i64([int(kept)]))[:, 0]
    total, offset = int(counts.sum()), int(counts[:rank].sum())
    r0, r1 = center_rank_window(total, max_size)
    lr0 = min(max(r0 - offset, 0), int(kept))
    lr1 = min(max(r1 - offset, 0), int(kept))
    w = np.ascontiguousarray(window_stats(lr0, lr1), dtype=np.float64)
    parts = np.asarray(allgather_i64(w.view(np.int64))).view(np.float64)
    g = np.array([parts[:, 0].sum(), parts[:, 1].min(), parts[:, 2].max(), 0.0, 0.0])
    for q in range(world):  # rank order, so every rank (and every world size's replay) folds identically
        g[3] += parts[q, 3]
        g[4] += parts[q, 4]
    st = center_stats_from_window(total, r0, r1, g)
    edges = center_bin_edges(st)
    if edges is None:
        return None
    y = allreduce_sum_i64(np.ascontiguousarray(histogram(lr0, lr1, edges), dtype=np.int64))
    return pick_center_from_histogram(y, edges)


def detect_center_distributed(ctx, rank, world, sb: ShardBuffer, noise_mag, mod_type, d_qad, max_size=None):
    """afp_demod of the shard into ``d_qad`` + the capture-wide detect_center, every rank ending with the same center.
    Exchange (NCCL, a few hundred bytes + one histogram): kept-sample counts -> global rank window; per-rank window
    partials {count, min, max, sum, sumsq} folded in rank order (deterministic) -> bin edges; histogram all-reduce.
    The bin width comes from Σ/Σ², not numpy's float32 variance: the reference's None-ness, center within one bin width (DESIGN §6)."""
    from .device import DeviceArray
    lib = ctx.lib
    code = _lib.demod_mod_code(mod_type)
    kept = C.c_int64(0)
    ctx.check(lib.urh_afp_demod_tiles(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, float(noise_mag), code,
                                      C.c_void_p(d_qad.ptr), int(rank > 0), C.byref(kept)))

    def window_stats(lr0, lr1):
        w = np.zeros(5, dtype=np.float64)
        ctx.check(lib.urh_center_window_stats(ctx.handle, C.c_void_p(d_qad.ptr), sb.n, lr0, lr1, w.ctypes.data_as(C.c_void_p)))
        return w

    def histogram(lr0, lr1, edges):
        nbins = len(edges) - 1
        y = np.zeros(nbins, dtype=np.int64)
        ctx.check(lib.urh_center_histogram_tiles(ctx.handle, C.c_void_p(d_qad.ptr), sb.n, lr0, lr1, C.c_double(edges[0]),
                                                 C.c_double(edges[1] - edges[0]), nbins, y.ctypes.data_as(C.c_void_p)))
        return y

    def allreduce(y):
        y = np.ascontiguousarray(y, dtype=np.int64)
        ctx.check(lib.urh_nccl_allreduce_host_i64(ctx.handle, y.ctypes.data_as(C.c_void_p), len(y), 0))
        return y

    return center_protocol(rank, world, kept.value, window_stats, histogram, lambda v: nccl_allgather_wide(ctx, world, v), allreduce,
                           max_size)


def demod_center_digitize_distributed(ctx, rank, world, sb: ShardBuffer, global_offset, n_total, noise_mag, mod_type, tolerance,
                                      samples_per_symbol, d_qad, bits_per_symbol=1, center_spacing=0.1, max_size=None, fetch=True,
                                      host_iq=None, rows_out=None, chunk_samples=1 << 24):
    """BASELINE configs[1]/[4] on N GPUs: demod + capture-wide detect_center + digitize of ONE sharded capture, one library
    call per rank (urh_shard_demod_center_digitize).  Exchanges, all NCCL on the context stream with device buffers: kept
    counts (8 B), window partials (32 B), the histogram all-reduce, then the digitizer's three 16-byte all-gathers.
    The digitizer pass reads the shard's qad (4 B/sample) once the center is known.  -> (center, rows or count).
    ``host_iq``: this rank's shard in (pinned) host memory: it is streamed into ``sb.shard`` in chunks while the chunks that have
    landed are demodulated (the halo sample must already be in ``sb.halo``); ``rows_out``: pinned int64 buffer for the rows."""
    lib = ctx.lib
    code = _lib.demod_mod_code(mod_type)
    if bits_per_symbol == 1:
        center, state, k = C.c_double(0.0), C.c_int(0), C.c_int64(0)
        if host_iq is not None:
            ctx.check(lib.urh_shard_demod_center_digitize_host(ctx.handle, host_iq.ctypes.data_as(C.c_void_p), _lib.dtype_code(sb.dtype), sb.n,
                                                               int(rank > 0), float(noise_mag), code, int(tolerance), int(samples_per_symbol),
                                                               -1 if max_size is None else int(max_size), int(chunk_samples),
                                                               C.c_void_p(sb.shard.ptr), C.c_void_p(d_qad.ptr), int(global_offset), int(n_total),
                                                               C.byref(center), C.byref(state), C.byref(k)))
        else:
            ctx.check(lib.urh_shard_demod_center_digitize(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, int(rank > 0),
                                                          float(noise_mag), code, int(tolerance), int(samples_per_symbol),
                                                          -1 if max_size is None else int(max_size), C.c_void_p(d_qad.ptr), int(global_offset),
                                                          int(n_total), C.byref(center), C.byref(state), C.byref(k)))
        if state.value == 0:
            return None, (np.zeros((0, 2), dtype=np.int64) if fetch else 0)
        if state.value == 1:
            if not fetch:
                return float(center.value), int(k.value)
            if rows_out is not None and rows_out.dtype == np.int64 and rows_out.size >= 2 * k.value:
                rows = rows_out.reshape(-1)[: 2 * k.value].reshape(k.value, 2)
            else:
                rows = np.empty((k.value, 2), dtype=np.int64)
            if k.value:
                ctx.check(lib.urh_fetch_pulses(ctx.handle, rows.ctypes.data_as(C.c_void_p), k.value))
            return float(center.value), rows
        # state 2: a tie the device must not break (every rank sees the same histogram, so every rank lands here together)
    center = detect_center_distributed(ctx, rank, world, sb, noise_mag, mod_type, d_qad, max_size)
    if center is None:
        return None, (np.zeros((0, 2), dtype=np.int64) if fetch else 0)
    out = demod_digitize_distributed(ctx, rank, world, sb, global_offset, n_total, noise_mag, mod_type, float(center), tolerance,
                                     samples_per_symbol, bits_per_symbol, center_spacing, None, fetch, qad_source=d_qad)
    return center, out


def merge_shard_rows(parts):
    """concatenate per-shard pulse tables; equal states that meet at a shard edge are one pulse (pyx:475-476)"""
    out = []
    for rows in parts:
        rows = np.asarray(rows, dtype=np.int64).reshape(-1, 2)
        if len(rows) == 0:
            continue
        if out and out[-1][-1, 0] == rows[0, 0]:
            out[-1][-1, 1] += rows[0, 1]
            rows = rows[1:]
        if len(rows):
            out.append(rows.copy())
    return np.concatenate(out) if out else np.zeros((0, 2), dtype=np.int64)


def detect_noise_level_sharded(ctx, hx, sb: ShardBuffer, global_offset, n_total):
    """AutoInterpretation.detect_noise_level over the whole capture from the 100 global, end-aligned chunks: every chunk is reduced
    whole by the rank that holds its first sample, with the single-GPU slice partition, so every chunk sum is the single-GPU word at
    any world size.  A chunk that a shard edge cuts is completed from the following shards first (``fetch_range``).  Two NCCL
    all-reduces (sum, max) then add one owner's value to zeros; the reference's host logic decides."""
    from .ainterpretation import AutoInterpretation as AI

    if n_total <= 3:
        return 0
    chunksize, nchunks = AI._chunking(n_total)
    lo, hi = int(global_offset), int(global_offset) + sb.n
    bounds = [(int(a), int(b)) for a, b in hx.allgather((lo, hi))]

    def holder(i):
        return next(q for q, (a, b) in enumerate(bounds) if a <= i < b)

    sums = np.zeros(nchunks, dtype=np.float64)
    maxs = np.full(nchunks, -1.0, dtype=np.float64)
    for j in range(nchunks):
        # global chunk j covers [n_total-(j+1)*cs, n_total-j*cs)
        c0, c1 = n_total - (j + 1) * chunksize, n_total - j * chunksize
        owner = holder(c0)
        if c1 <= bounds[owner][1]:
            part = sb.shard[c0 - lo: c1 - lo] if hx.rank == owner else None
        else:
            part = fetch_range(ctx, hx.rank, bounds, sb.shard, c0, c1, owner)   # collective: every rank takes this branch
        if hx.rank != owner:
            continue
        s1, m1 = np.zeros(1), np.zeros(1)
        ctx.check(ctx.lib.urh_noise_chunk_stats_iq(ctx.handle, C.c_void_p(part.ptr), _lib.dtype_code(sb.dtype), chunksize, chunksize, 1,
                                                   s1.ctypes.data_as(C.c_void_p), m1.ctypes.data_as(C.c_void_p)))
        sums[j], maxs[j] = s1[0], m1[0]
    d_s = DeviceArray(ctx, (nchunks,), np.float64).set(sums)
    d_m = DeviceArray(ctx, (nchunks,), np.float64).set(maxs)
    ctx.check(ctx.lib.urh_nccl_allreduce_f64(ctx.handle, C.c_void_p(d_s.ptr), nchunks, 0))
    ctx.check(ctx.lib.urh_nccl_allreduce_f64(ctx.handle, C.c_void_p(d_m.ptr), nchunks, 1))
    return AI._noise_from_chunk_stats(n_total, chunksize, d_s.get(), d_m.get(), np.float64)


# ---- AutoInterpretation.estimate over a sharded capture (BASELINE configs[4]) ------------------------------------------------------
def segment_messages_sharded(ctx, hx, d_mag, global_offset, n_total, noise_threshold):
    """segment_messages_from_magnitudes (auto_interpretation.pyx:55-111) of a capture whose magnitudes are spread over the ranks:
    every rank runs the dense pass over its shard; the closing-run summaries are folded (``fold_carry``) so that runs crossing a
    shard edge count their samples on both sides; the run tables (a few entries per message) are concatenated in rank order and
    every rank runs the reference's two-state machine on them.  Returns the same list of (start, end) on every rank."""
    lib = ctx.lib
    n_local = len(d_mag)
    summary = (C.c_int64 * 4)()
    ctx.check(lib.urh_segment_shard_pass(ctx.handle, C.c_void_p(d_mag.ptr), int(d_mag.dtype == np.float64), n_local,
                                         float(noise_threshold), summary))
    every = hx.allgather((int(summary[0]), int(summary[1]), int(summary[2]), int(summary[3])))
    carries = fold_carry([(c, l, w) for c, l, w, _ in every])
    carry = carries[hx.rank]
    count = C.c_int64(0)
    ctx.check(lib.urh_shard_candidates(ctx.handle, int(carry is not None), carry[0] if carry else 0, carry[1] if carry else 0,
                                       int(global_offset), C.byref(count), None, None, None))
    pos = np.empty(count.value, dtype=np.int64)
    cls = np.empty(count.value, dtype=np.int16)
    if count.value:
        ctx.check(lib.urh_fetch_candidates(ctx.handle, pos.ctypes.data_as(C.c_void_p), cls.ctypes.data_as(C.c_void_p), count.value))
    tables = hx.allgather((pos, cls))
    pos_all = np.ascontiguousarray(np.concatenate([t[0] for t in tables]))
    cls_all = np.ascontiguousarray(np.concatenate([t[1] for t in tables]))
    # the run that ends the capture: fold every shard's closing run
    last_cls, last_len = None, 0
    for c, l, w, _ in every:
        if last_cls is not None and w and c == last_cls:
            last_len += l
        else:
            last_cls, last_len = c, l
    cap = max(16, len(pos_all) + 2)
    seg = np.empty((cap, 2), dtype=np.int64)
    k = C.c_int64(0)
    ctx.check(lib.urh_segments_from_runs(pos_all.ctypes.data_as(C.c_void_p), cls_all.ctypes.data_as(C.c_void_p), len(pos_all), int(every[0][3]),
                                         int(last_cls), int(last_len), int(n_total), seg.ctypes.data_as(C.c_void_p), cap, C.byref(k)))
    return [(int(a), int(b)) for a, b in seg[: k.value]]


def fetch_range(ctx, rank, bounds, d_local, g0, g1, owner):
    """Collective: every rank calls it with the same (g0, g1, owner).  `d_local` is this rank's shard (1-D or (n, 2) DeviceArray) of
    a capture cut at `bounds` [(start, end) per rank].  Returns on `owner` a DeviceArray with elements [g0, g1) of the capture
    (its own part copied, the other parts received over NCCL); None elsewhere."""
    lib = ctx.lib
    item = d_local.nbytes // max(1, len(d_local))
    out = None
    if rank == owner:
        shape = (g1 - g0,) + tuple(d_local.shape[1:])
        out = DeviceArray(ctx, shape, d_local.dtype)
    for q, (a, b) in enumerate(bounds):
        lo, hi = max(a, g0), min(b, g1)
        if lo >= hi:
            continue
        nbytes = (hi - lo) * item
        if q == owner:
            if rank == owner:
                ctx.check(lib.urh_memcpy_d2d(ctx.handle, C.c_void_p(out.ptr + (lo - g0) * item), C.c_void_p(d_local.ptr + (lo - a) * item), nbytes))
        elif rank == q:
            ctx.check(lib.urh_nccl_sendrecv(ctx.handle, C.c_void_p(d_local.ptr + (lo - a) * item), nbytes, owner, None, 0, -1))
        elif rank == owner:
            ctx.check(lib.urh_nccl_sendrecv(ctx.handle, None, 0, -1, C.c_void_p(out.ptr + (lo - g0) * item), nbytes, q))
    return out


def estimate_sharded(ctx, hx, sb: ShardBuffer, bounds, n_total, noise=None, modulation=None):
    """AutoInterpretation.estimate (AutoInterpretation.py:373-471) of ONE capture sharded by contiguous sample range: the same dict
    on every rank, equal to the single-GPU / reference result.
      noise       global end-aligned chunk statistics, NCCL all-reduce (detect_noise_level_sharded)
      messages    sharded segmentation with run carry (segment_messages_sharded)
      modulation  detect_modulation on the first 100 messages, each on the rank that owns its start
      demod       ASK / FSK with the 1-sample halo; PSK with the speculative Costas loop over shards (afp_demod_psk_sharded)
      parameters  detect_center / plateau lengths / tolerance / bit length per message on the owning rank (a message that
                  straddles a shard edge is completed over NCCL), gathered and reduced exactly as the reference does."""
    from .ainterpretation import AutoInterpretation as AI
    from .cythonext import auto_interpretation as c_ai
    from .cythonext import signal_functions as sf
    from .cythonext import util

    rank, world = hx.rank, hx.world
    lo, hi = bounds[rank]
    d_mag = util.get_magnitudes(sb.shard)
    if noise is None:
        noise = detect_noise_level_sharded(ctx, hx, sb, lo, n_total)
    message_indices = segment_messages_sharded(ctx, hx, d_mag, lo, n_total, noise)
    d_mag.free()

    def owner_of(start):
        for q, (a, b) in enumerate(bounds):
            if a <= start < b:
                return q
        return world - 1

    def message_slice(d_shard, start, end):
        """[start, end) of the capture on the rank owning `start` (collective when the message leaves that rank's shard)"""
        own = owner_of(start)
        a, b = bounds[own]
        if end <= b:
            return (d_shard[start - a: end - a] if rank == own else None), own
        return fetch_range(ctx, rank, bounds, d_shard, start, end, own), own

    if modulation is None:
        found_local = []
        for idx, (start, end) in enumerate(message_indices[0:100]):
            part, own = message_slice(sb.shard, start, end)
            if rank == own:
                from .signalprocessing.IQArray import IQArray
                mod = AI.detect_modulation(IQArray(np.ascontiguousarray(part.get()), _owned=True).as_complex64())
                if mod is not None:
                    found_local.append((idx, mod))
        found = sorted(x for part in hx.allgather(found_local) for x in part)
        modulation = AI.most_common([m for _, m in found]) if found else None
    if modulation is None:
        return None
    if modulation == "OOK":
        message_indices = AI.merge_message_segments_for_ook(message_indices)
    d_qad = DeviceArray(ctx, (hi - lo,), np.float32)
    if modulation == "PSK":
        afp_demod_psk_sharded(ctx, rank, world, sb, noise, 2, 0.1, d_qad)
    else:
        mt = "ASK" if modulation in ("OOK", "ASK") else "FSK"
        kept = C.c_int64(0)
        ctx.check(ctx.lib.urh_afp_demod_tiles(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, float(noise),
                                              _lib.demod_mod_code(mt), C.c_void_p(d_qad.ptr), int(rank > 0), C.byref(kept)))
    local = []   # (message index, center, bit_length or None, tolerance or None)
    for idx, (start, end) in enumerate(message_indices):
        msg, own = message_slice(d_qad, int(start), int(end))
        if rank != own:
            continue
        center = AI.detect_center(msg)
        if center is None:
            continue
        plateau_lengths = c_ai.get_plateau_lengths(msg, center, percentage=25)
        tolerance = AI.estimate_tolerance_from_plateau_lengths(plateau_lengths)
        tol_entry = None
        if tolerance is None:
            tolerance = 0
        else:
            tol_entry = tolerance
        merged = AI.merge_plateau_lengths(plateau_lengths, tolerance=tolerance)
        bit_entry = None
        if len(merged) >= 2:
            bit_length = AI.get_bit_length_from_plateau_lengths(merged)
            if bit_length > tolerance + 1:
                bit_entry = (float(center), bit_length)
        local.append((idx, tol_entry, bit_entry))
    rows = sorted(x for part in hx.allgather(local) for x in part)
    tolerances = [t for _, t, _ in rows if t is not None]
    centers = [b[0] for _, _, b in rows if b is not None]
    bit_lengths = [b[1] for _, _, b in rows if b is not None]
    if modulation in ("OOK", "ASK"):
        center = AI.min_without_outliers(np.array(centers), z=2)
        if center is None:
            return None
    elif len(centers) > 0:
        center = np.mean(centers)
    else:
        return None
    bit_length = AI.get_most_frequent_value(bit_lengths)
    if bit_length is None:
        return None
    try:
        tolerance = np.percentile(tolerances, 50)
    except IndexError:
        tolerance = max(1, int(0.05 * bit_length))
    return {"modulation_type": "ASK" if modulation == "OOK" else modulation, "bit_length": bit_length, "center": center,
            "tolerance": int(tolerance), "noise": noise}


# ---- filters and spectrogram over shards (DESIGN.md §6, "Filters and spectrogram over shards") -----------------------------------------
# Every band-pass / FIR output and every spectrogram frame depends on its own input window only, with a fixed accumulation order, so a
# rank that holds that window (its shard plus halos copied from its neighbours) computes the single-GPU words bit for bit.  The plans
# are pure host logic, computed identically on every rank from `bounds`; they raise ValueError before any collective, so every rank
# raises alike and none is left waiting inside NCCL.
def _check_bounds(bounds):
    bounds = [(int(a), int(b)) for a, b in bounds]
    if not bounds or bounds[0][0] != 0 or any(b <= a for a, b in bounds) or any(bounds[q][1] != bounds[q + 1][0] for q in range(len(bounds) - 1)):
        raise ValueError("bounds must cut the capture into contiguous, non-empty shards starting at sample 0")
    return bounds


def _check_halos(bounds, halos, what):
    """halos[r] = (left, right): rank r - 1 supplies `left` samples and rank r + 1 `right` samples, from their own shards only"""
    last = len(bounds) - 1
    for r, (left, right) in enumerate(halos):
        if left and (r == 0 or bounds[r - 1][1] - bounds[r - 1][0] < left):
            raise ValueError("%s: shard %d (%d samples) is shorter than the %d-sample halo shard %d needs"
                             % (what, r - 1, bounds[r - 1][1] - bounds[r - 1][0] if r else 0, left, r))
        if right and (r == last or bounds[r + 1][1] - bounds[r + 1][0] < right):
            raise ValueError("%s: shard %d (%d samples) is shorter than the %d-sample halo shard %d needs"
                             % (what, r + 1, bounds[r + 1][1] - bounds[r + 1][0] if r < last else 0, right, r))


def bandpass_plan(n_total, m, bounds):
    """Filter.apply_bandpass_filter of an m-tap filter over a capture cut at `bounds` -> [(L, R, offset)] per rank: rank r convolves the
    window x[g0 - L, g1 + R) with urh_convolve_c128 at `offset` for g1 - g0 outputs.  Both of the reference's branches (np.convolve
    'same' and the centred FFT crop) give full_convolution[(m - 1) // 2 + k], k < N, for a filter no longer than the capture (odd on
    the FFT branch); the inputs where the single-GPU function changes the length or returns nothing raise ValueError."""
    bounds = _check_bounds(bounds)
    n_total, m = int(n_total), int(m)
    if n_total != bounds[-1][1]:
        raise ValueError("bounds do not cover the %d-sample capture" % n_total)
    if m < 1:
        raise ValueError("band-pass: empty filter")
    if n_total < m:
        raise ValueError("band-pass: the capture (%d samples) is shorter than the %d-tap filter: np.convolve(..., 'same') returns %d samples"
                         % (n_total, m, m))
    if not m < 8 * math.log(math.sqrt(n_total)):   # Filter.apply_bandpass_filter's branch rule: the FFT convolution
        if m <= 2:
            raise ValueError("band-pass: the FFT convolution of a %d-tap filter returns an empty array" % m)
        if m % 2 == 0:
            raise ValueError("band-pass: the FFT convolution of an even %d-tap filter returns %d samples" % (m, n_total + 1))
    half = (m - 1) // 2
    last = len(bounds) - 1
    plan = []
    for r in range(len(bounds)):
        left = 0 if r == 0 else m - 1 - half
        right = 0 if r == last else half
        plan.append((left, right, left + half))
    _check_halos(bounds, [(left, right) for left, right, _ in plan], "band-pass")
    return plan


def fir_plan(n_total, m, bounds):
    """Filter.apply_fir_filter (causal fir_filter) over a capture cut at `bounds` -> the history length per rank: rank r > 0 reads the
    previous shard's last m - 1 samples instead of the zero initial state (urh_fir_filter_shard)."""
    bounds = _check_bounds(bounds)
    if int(n_total) != bounds[-1][1]:
        raise ValueError("bounds do not cover the %d-sample capture" % n_total)
    hist = [0 if r == 0 else max(0, int(m) - 1) for r in range(len(bounds))]
    _check_halos(bounds, [(h, 0) for h in hist], "FIR")
    return hist


def frame_plan(n_total, window_size, hop, bounds):
    """Spectrogram frames over a capture cut at `bounds` -> [(first_frame, frames, R)] per rank.  Frame f (of Spectrogram._num_frames)
    belongs to the rank holding sample f * hop; R is what that rank's last frame reads past its shard (from the next one)."""
    bounds = _check_bounds(bounds)
    n_total, W, hop = int(n_total), int(window_size), int(hop)
    if n_total != bounds[-1][1]:
        raise ValueError("bounds do not cover the %d-sample capture" % n_total)
    if W <= 0 or hop <= 0:
        raise ValueError("spectrogram: bad window size %d / hop %d" % (W, hop))
    frames = max(1, (max(n_total, W) - W) // hop + 1)
    plan = []
    for g0, g1 in bounds:
        f0 = -(-g0 // hop)
        f1 = min(frames, -(-g1 // hop))
        nf = max(0, f1 - f0)
        right = max(0, min(n_total, (f1 - 1) * hop + W) - g1) if nf else 0
        plan.append((f0, nf, right))
    _check_halos(bounds, [(0, right) for _, _, right in plan], "spectrogram")
    return plan


def segment_plan(n_total, window_size, hop, bounds, max_lines=None):
    """The image segments of Spectrogram.create_image_segments over a capture cut at `bounds` -> (segments, owned, rights):
    segments = Spectrogram.segment_bounds of the whole capture, owned[r] = indices of the segments that start in shard r (their tail
    comes from the next shard), rights[r] = how far the last of them reaches past shard r."""
    from .signalprocessing.Spectrogram import Spectrogram

    bounds = _check_bounds(bounds)
    n_total = int(n_total)
    if n_total != bounds[-1][1]:
        raise ValueError("bounds do not cover the %d-sample capture" % n_total)
    if int(window_size) <= 0 or int(hop) <= 0:
        raise ValueError("spectrogram: bad window size %d / hop %d" % (window_size, hop))
    segments = Spectrogram.segment_bounds_of(n_total, int(window_size), int(hop),
                                             Spectrogram.MAX_LINES_PER_VIEW if max_lines is None else int(max_lines))
    owned = [[i for i, (s, _, _) in enumerate(segments) if g0 <= s < g1] for g0, g1 in bounds]
    rights = [max([0] + [segments[i][1] - g1 for i in mine]) for mine, (_, g1) in zip(owned, bounds)]
    _check_halos(bounds, [(0, right) for right in rights], "spectrogram images")
    return segments, owned, rights


def dc_exact_handover(rank, world, chain, allgather):
    """The serial float32 column sums of a capture sharded over the ranks: rank r continues the chain from the two accumulators rank
    r - 1 ended with (``chain(carry) -> float32[2]``), in rank order; ``allgather(float32[2]) -> [world, 2]``.  Every rank returns the
    sums of the whole capture, bit for bit numpy's serial chain."""
    carry = np.zeros(2, dtype=np.float32)
    for turn in range(world):
        mine = np.asarray(chain(carry), dtype=np.float32) if turn == rank else np.zeros(2, dtype=np.float32)
        carry = np.asarray(allgather(mine), dtype=np.float32).reshape(world, 2)[turn].copy()
    return carry


def dc_fold_double(parts, n_total):
    """float32 mean from per-rank double column sums [world, 2], added in rank order (the double regime of the DC correction)"""
    s = np.zeros(2, dtype=np.float64)
    for q in range(len(parts)):
        s = s + np.asarray(parts[q], dtype=np.float64)
    return (s / float(n_total)).astype(np.float32)


def exchange_halos(ctx, hx, sb: ShardBuffer, halos=None):
    """Rank r receives halos[r][0] samples of rank r - 1's tail into the samples right before its shard and halos[r][1] of rank r + 1's
    head right after it: two grouped NCCL send/recv on the context stream, device to device.  ``halos``: [(left, right)] per rank, the
    same on every rank (by default every rank's (halo_len, right_len))."""
    rank, world = hx.rank, hx.world
    if halos is None:
        halos = hx.allgather((sb.halo_len, sb.right_len))
    left = int(halos[rank][0]) if rank > 0 else 0
    right = int(halos[rank][1]) if rank < world - 1 else 0
    to_next = int(halos[rank + 1][0]) if rank + 1 < world else 0    # my tail -> rank + 1
    to_prev = int(halos[rank - 1][1]) if rank > 0 else 0            # my head -> rank - 1
    assert left <= sb.halo_len and right <= sb.right_len and to_next <= sb.n and to_prev <= sb.n
    item = 2 * sb.dtype.itemsize
    lib = ctx.lib
    if to_next or left:
        ctx.check(lib.urh_nccl_sendrecv(ctx.handle, C.c_void_p(sb.shard.ptr + (sb.n - to_next) * item), to_next * item, rank + 1 if to_next else -1,
                                        C.c_void_p(sb.shard.ptr - left * item), left * item, rank - 1 if left else -1))
    if to_prev or right:
        ctx.check(lib.urh_nccl_sendrecv(ctx.handle, C.c_void_p(sb.shard.ptr), to_prev * item, rank - 1 if to_prev else -1,
                                        C.c_void_p(sb.right.ptr), right * item, rank + 1 if right else -1))


def _with_room(ctx, sb: ShardBuffer, left, right):
    """`sb` if it has room for the halos, else a copy of its shard in a buffer that has"""
    if sb.halo_len >= left and sb.right_len >= right:
        return sb
    out = ShardBuffer(ctx, sb.n, sb.dtype, halo=max(left, sb.halo_len), right=max(right, sb.right_len))
    ctx.check(ctx.lib.urh_memcpy_d2d(ctx.handle, C.c_void_p(out.shard.ptr), C.c_void_p(sb.shard.ptr), sb.shard.nbytes))
    return out


def _output_halos(ctx, bounds, world, out_halo):
    """the left halo of a filtered shard buffer: what the sharded demodulators read before the shard (default: the Costas warm-up)"""
    h = costas_halo(ctx) if out_halo is None else int(out_halo)
    halos = [(h if r else 0, 0) for r in range(world)]
    _check_halos(bounds, halos, "filter output")
    return h, halos


def _float_shard(sb, what):
    if sb.dtype != np.float32:
        raise ValueError("%s: the shards must be complex64 samples (float32 (n, 2))" % what)


def apply_bandpass_filter_sharded(ctx, hx, sb: ShardBuffer, bounds, f_low, f_high, filter_bw=0.08, out_halo=None) -> ShardBuffer:
    """Filter.apply_bandpass_filter (Filter.py:84-101) of a capture sharded over the ranks, bit for bit the single-GPU result.  Rank r
    receives the filter-length halos from its neighbours (``bandpass_plan``) and convolves its window; the output comes back as a
    ShardBuffer whose left halo already holds the previous shard's filtered tail, so demod_center_digitize_distributed /
    afp_demod_psk_sharded take it directly."""
    from .signalprocessing.Filter import Filter

    bounds = _check_bounds(bounds)
    rank, world = hx.rank, hx.world
    _float_shard(sb, "band-pass")
    h = np.ascontiguousarray(Filter.bandpass_taps(f_low, f_high, filter_bw), dtype=np.complex128)
    plan = bandpass_plan(bounds[-1][1], len(h), bounds)
    out_h, out_halos = _output_halos(ctx, bounds, world, out_halo)
    left, right, offset = plan[rank]
    src = _with_room(ctx, sb, left, right)
    exchange_halos(ctx, hx, src, [(a, b) for a, b, _ in plan])
    win = src.window(left, right)
    d_t = to_device(h.view(np.float64), ctx)
    out = ShardBuffer(ctx, sb.n, np.float32, halo=out_h)
    ctx.check(ctx.lib.urh_convolve_c128(ctx.handle, C.c_void_p(win.ptr), len(win), C.c_void_p(d_t.ptr), len(h), int(offset), sb.n,
                                        C.c_void_p(out.shard.ptr)))
    if not len(h) < 8 * math.log(math.sqrt(bounds[-1][1])):
        # the FFT branch: one non-finite sample anywhere in the capture makes every output NaN + NaN j (Filter._convolve_full_slice)
        flag = to_device(np.zeros(1, np.int32), ctx)
        ctx.check(ctx.lib.urh_nonfinite_flag(ctx.handle, C.c_void_p(out.shard.ptr), sb.n, C.c_void_p(flag.ptr)))
        if any(int(f) for f in hx.allgather(int(flag.get()[0]))):
            flag = to_device(np.ones(1, np.int32), ctx)
            ctx.check(ctx.lib.urh_nan_fill_if(ctx.handle, C.c_void_p(out.shard.ptr), sb.n, C.c_void_p(flag.ptr)))
    exchange_halos(ctx, hx, out, out_halos)
    ctx.sync()
    return out


def fir_filter_sharded(ctx, hx, sb: ShardBuffer, bounds, taps, out_halo=None) -> ShardBuffer:
    """Filter.apply_fir_filter (fir_filter, signal_functions.pyx:513-525) of a capture sharded over the ranks: rank r > 0 filters its
    shard with the previous shard's last m - 1 samples as history (urh_fir_filter_shard), bit for bit the single-GPU result."""
    bounds = _check_bounds(bounds)
    rank, world = hx.rank, hx.world
    _float_shard(sb, "FIR")
    taps = np.ascontiguousarray(np.asarray(taps, dtype=np.complex64))
    hist = fir_plan(bounds[-1][1], len(taps), bounds)
    out_h, out_halos = _output_halos(ctx, bounds, world, out_halo)
    src = _with_room(ctx, sb, hist[rank], 0)
    exchange_halos(ctx, hx, src, [(a, 0) for a in hist])
    d_t = to_device(taps.view(np.float32) if len(taps) else np.zeros(2, np.float32), ctx)
    out = ShardBuffer(ctx, sb.n, np.float32, halo=out_h)
    ctx.check(ctx.lib.urh_fir_filter_shard(ctx.handle, C.c_void_p(src.shard.ptr), sb.n, int(hist[rank] > 0), C.c_void_p(d_t.ptr), len(taps),
                                           C.c_void_p(out.shard.ptr)))
    exchange_halos(ctx, hx, out, out_halos)
    ctx.sync()
    return out


def dc_correction_sharded(ctx, hx, sb: ShardBuffer, bounds, out_halo=None) -> ShardBuffer:
    """Filter.dc_correction (Filter.py:31-33) of a capture sharded over the ranks.
      float32, N <= Filter.EXACT_DC_MAX: numpy's serial float32 column chain handed from rank to rank (``dc_exact_handover``), then
                 sum / N in float32 on every rank: bit for bit the single-GPU result;
      float32, larger N: per-rank double column sums, all-gathered and added in rank order (``dc_fold_double``), mean = float32(sum / N);
      integer captures: exact int64 column sums added over the ranks, mean = sum / N in double; a float64 result, bit for bit."""
    from .signalprocessing.Filter import Filter

    bounds = _check_bounds(bounds)
    rank, world = hx.rank, hx.world
    n_total = bounds[-1][1]
    lib = ctx.lib
    if sb.dtype == np.float32:
        out_h, out_halos = _output_halos(ctx, bounds, world, out_halo)
        if n_total <= Filter.EXACT_DC_MAX:
            def chain(carry):
                c = np.ascontiguousarray(carry, dtype=np.float32)
                s = np.zeros(2, dtype=np.float64)
                ctx.check(lib.urh_dc_column_sums(ctx.handle, C.c_void_p(sb.shard.ptr), sb.n, 1, c.ctypes.data_as(C.c_void_p),
                                                 s.ctypes.data_as(C.c_void_p)))
                return s.astype(np.float32)   # float32 accumulators carried in doubles: exact

            def allgather(pair):
                every = nccl_allgather_wide(ctx, world, np.ascontiguousarray(pair, dtype=np.float32).view(np.int64))
                return np.ascontiguousarray(every).view(np.float32).reshape(world, 2)
            mean = dc_exact_handover(rank, world, chain, allgather) / np.float32(n_total)
        else:
            s = np.zeros(2, dtype=np.float64)
            ctx.check(lib.urh_dc_column_sums(ctx.handle, C.c_void_p(sb.shard.ptr), sb.n, 0, None, s.ctypes.data_as(C.c_void_p)))
            every = nccl_allgather_wide(ctx, world, s.view(np.int64))
            mean = dc_fold_double(np.ascontiguousarray(every).view(np.float64).reshape(world, 2), n_total)
        out = ShardBuffer(ctx, sb.n, np.float32, halo=out_h)
        ctx.check(lib.urh_dc_subtract(ctx.handle, C.c_void_p(sb.shard.ptr), sb.n, float(mean[0]), float(mean[1]), C.c_void_p(out.shard.ptr)))
        exchange_halos(ctx, hx, out, out_halos)
    elif sb.dtype in (np.int8, np.uint8, np.int16, np.uint16):
        s = np.zeros(2, dtype=np.int64)
        ctx.check(lib.urh_dc_int_column_sums(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, s.ctypes.data_as(C.c_void_p)))
        every = nccl_allgather_wide(ctx, world, s)
        mean = [float(sum(int(v) for v in every[:, c])) / float(n_total) for c in (0, 1)]
        out = ShardBuffer(ctx, sb.n, np.float64, halo=0)
        ctx.check(lib.urh_dc_int_subtract(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(sb.dtype), sb.n, mean[0], mean[1],
                                          C.c_void_p(out.shard.ptr)))
    else:
        raise ValueError("dc_correction expects an (n, 2) capture of int8/uint8/int16/uint16/float32")
    ctx.sync()
    return out


def filter_work_sharded(ctx, hx, sb: ShardBuffer, bounds, filt, out_halo=None) -> ShardBuffer:
    """Filter.work (Filter.py:30-33) of a capture sharded over the ranks: the DC correction or the FIR filter of ``filt``"""
    from .signalprocessing.Filter import FilterType

    if filt.filter_type == FilterType.dc_correction:
        return dc_correction_sharded(ctx, hx, sb, bounds, out_halo)
    return fir_filter_sharded(ctx, hx, sb, bounds, filt.taps, out_halo)


def spectrogram_db_sharded(ctx, hx, sb: ShardBuffer, bounds, window_size=1024, overlap_factor=0.5, window_function=np.hanning):
    """Spectrogram.calculate_spectrogram (Spectrogram.py:156-162) of a capture sharded over the ranks -> (first_frame, DeviceArray
    [frames, W]): the rows of the single-GPU dB map this rank owns (``frame_plan``), bit for bit."""
    bounds = _check_bounds(bounds)
    rank = hx.rank
    _float_shard(sb, "spectrogram")
    W = int(window_size)
    hop = W - int(overlap_factor * W)
    plan = frame_plan(bounds[-1][1], W, hop, bounds)
    f0, nf, right = plan[rank]
    src = _with_room(ctx, sb, 0, right)
    exchange_halos(ctx, hx, src, [(0, r) for _, _, r in plan])
    out = DeviceArray(ctx, (nf, W), np.float32)
    if nf:
        win = src.window(0, right)[f0 * hop - bounds[rank][0]:]
        d_w = to_device(np.ascontiguousarray(window_function(W), dtype=np.float64), ctx)
        ctx.check(ctx.lib.urh_spectrogram_db(ctx.handle, C.c_void_p(win.ptr), len(win), W, hop, C.c_void_p(d_w.ptr), nf, C.c_void_p(out.ptr)))
    ctx.sync()
    return f0, out


def spectrogram_image_segments_sharded(ctx, hx, sb: ShardBuffer, bounds, window_size=1024, overlap_factor=0.5, window_function=np.hanning,
                                       colormap=None, data_min=-140, data_max=10, transpose=False):
    """Spectrogram.create_image_segments (Spectrogram.py:183-190) of a capture sharded over the ranks -> [(segment_index, image)] of the
    segments that start in this rank's shard (``segment_plan``), each a uint8 DeviceArray [W][frames][4] (transpose: [frames][W][4], the
    layout of create_spectrogram_image(start, end, transpose=True)), bit for bit the single-GPU images."""
    from .signalprocessing.Spectrogram import Spectrogram

    bounds = _check_bounds(bounds)
    rank = hx.rank
    _float_shard(sb, "spectrogram images")
    cmap = Spectrogram._colormap(colormap)
    spec = Spectrogram(None, window_size=int(window_size), overlap_factor=overlap_factor, window_function=window_function)
    spec.data_min, spec.data_max = data_min, data_max
    segments, owned, rights = segment_plan(bounds[-1][1], spec.window_size, spec.hop_size, bounds, spec.MAX_LINES_PER_VIEW)
    right = rights[rank]
    src = _with_room(ctx, sb, 0, right)
    exchange_halos(ctx, hx, src, [(0, r) for r in rights])
    mine = owned[rank]
    if not mine:
        ctx.sync()
        return []
    g0 = bounds[rank][0]
    win = src.window(0, right)
    out, shapes = spec._images(win, len(win), [(segments[i][0] - g0, segments[i][1] - segments[i][0]) for i in mine], transpose, cmap, ctx)
    ctx.sync()
    return list(zip(mine, spec._split(out, shapes, True)))
