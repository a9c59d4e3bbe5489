// grab_pulse_lens after the dense pass, entirely at TILE level (signal_functions.pyx:455-495; DESIGN.md 4.2).
//
// The dense pass leaves per tile a 16-byte summary and the staged interior candidates.  Everything that used to
// work on the gathered candidate table (gather, fire flags, three int64 scans over ~n/100 entries, three scalar
// read-backs) is restated on the tile table (n/2048 entries) as three look-back scans and one row kernel:
//
//   A  run carry           exclusive scan of {class, length, whole?} of each tile's closing run  -> carry[t]
//   B  candidates          per tile: head candidate from carry[t] (+ the carry of the preceding shards), number of
//                          candidates, class of the last one; scan -> class of the candidate preceding the tile.  The
//                          same walk over the staged words leaves the tile's firings apart from its first candidate's
//                          (a candidate fires iff its class differs from the one before it) -> fire[t]
//   C  firings             per tile: fire[t] plus the first candidate's firing against the preceding class (O(1));
//                          scan -> row offset, previous firing
//   D  rows                per tile: walk again, write (state, length) rows at the tile's row offset; the last
//                          tile appends the tail row (pyx:485-493) and the row count
// B walks one THREAD per tile (it reads the staging row for the last class anyway, and counting needs no more than that).
// D runs one WARP per 32 consecutive tiles: the lanes take 32 candidates of a tile at once, the firings come from a ballot,
// and the rows of one chunk land at consecutive addresses.  The first 32 staged words of eight tiles are loaded before the
// first of them is walked.
//
// One read-back (row count) ends the call.  Rows go straight into the context's pulse buffer, sized optimistically;
// an overflow only repeats stage D.  ASK (short pauses relabelled, pyx:471-473, so equal neighbours can meet) runs a
// fourth scan that merges equal neighbours.
//
// Sharded captures (SURVEY 8e): between the stages every rank publishes its scan total (16 bytes) with an NCCL
// all-gather ON THE CONTEXT STREAM into device memory and a one-thread kernel folds the totals of the preceding
// ranks; the host never waits between the stages.
#include "sparse.cuh"
#include "tilescan.cuh"

#include <limits.h>

#define CLS_NONE INT_MIN

// ---- scan elements --------------------------------------------------------------------------------------------------
struct __align__(16) CandAgg {
    int64_t cnt;       // candidates
    int32_t last_cls;  // class of the last candidate (CLS_NONE: no candidate in the span)
    int32_t pad;
};
struct CandOp {
    __device__ __forceinline__ CandAgg operator()(const CandAgg& a, const CandAgg& b) const {
        CandAgg r;
        r.cnt = a.cnt + b.cnt;
        r.last_cls = (b.last_cls != CLS_NONE) ? b.last_cls : a.last_cls;
        r.pad = 0;
        return r;
    }
};
struct __align__(16) FireAgg {
    int64_t fired;     // firings
    int64_t last_pos;  // global position of the last firing (-1: none in the span)
};
struct FireOp {
    __device__ __forceinline__ FireAgg operator()(const FireAgg& a, const FireAgg& b) const {
        FireAgg r;
        r.fired = a.fired + b.fired;
        r.last_pos = (b.last_pos >= 0) ? b.last_pos : a.last_pos;
        return r;
    }
};

// ---- A ---------------------------------------------------------------------------------------------------------------
struct ScanRunCarry : TileRuns {
    RunCarry* carry;
    __device__ __forceinline__ void post(int64_t t, const RunCarry& excl, const RunCarry&) const { carry[t] = excl; }
};

// ---- B ---------------------------------------------------------------------------------------------------------------
// The tile's candidates apart from the class that precedes them: its first candidate, and the firings after it (each candidate
// against the one before it inside the tile).  Stage C decides the first one's firing once the preceding class is known.
struct __align__(16) TileFire {
    int32_t first_cls;   // class of the first candidate (CLS_NONE: the tile has none)
    int32_t first_rel;   // its tile-relative position
    int32_t fired;       // firings among the later candidates
    int32_t last_rel;    // tile-relative position of the last of those (-1: none)
};
struct ScanCandidates {
    const UrhTileSummary* tiles;
    const uint32_t* staging;
    int stage_cap;
    const RunCarry* carry;
    const RunCarry* xcarry;   // device: the run that ends right before this shard (nullptr: unsharded)
    int tol;
    int32_t* head_rel;
    int32_t* prev_cls;
    TileFire* fire;
    __device__ __forceinline__ CandAgg load(int64_t t) const {
        const UrhTileSummary s = tiles[t];
        RunCarry c = carry[t];
        if (xcarry) c = RunCarryOp()(*xcarry, c);
        int64_t start_len = 0;
        if (!(c.flags & 2) && c.cls == s.first_cls) start_len = c.len;
        int32_t rel = -1;
        if (start_len <= tol && (int64_t)tol < start_len + s.head_len) rel = (int32_t)(tol - start_len);
        head_rel[t] = rel;
        TileFire f;
        f.first_cls = CLS_NONE; f.first_rel = -1; f.fired = 0; f.last_rel = -1;
        int prev = CLS_NONE;
        if (rel >= 0) {
            prev = s.first_cls;
            f.first_cls = prev;
            f.first_rel = rel;
        }
        // the staged words (~20 per tile on the bench capture), four loads in flight
        const uint32_t* st = staging + t * (int64_t)stage_cap;
        for (int j = 0; j < s.ncand; j += 4) {
            uint32_t w[4];
#pragma unroll
            for (int u = 0; u < 4; u++) w[u] = (j + u < s.ncand) ? st[j + u] : 0u;
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (j + u < s.ncand) {
                    const int cl = (int)(w[u] & 0xffffu) - 1;
                    const int p = (int)(w[u] >> 16);
                    if (prev == CLS_NONE) {
                        f.first_cls = cl;
                        f.first_rel = p;
                    } else if (cl != prev) {
                        f.fired++;
                        f.last_rel = p;
                    }
                    prev = cl;
                }
            }
        }
        fire[t] = f;
        CandAgg r;
        r.cnt = (int64_t)s.ncand + (rel >= 0 ? 1 : 0);
        r.last_cls = prev;
        r.pad = 0;
        return r;
    }
    __device__ __forceinline__ void post(int64_t t, const CandAgg& excl, const CandAgg&) const { prev_cls[t] = excl.last_cls; }
};

// ---- C ---------------------------------------------------------------------------------------------------------------
struct ScanFirings {
    const TileFire* fire;
    const int32_t* prev_cls;
    const int16_t* d_prev0;   // device: class of the candidate preceding the shard (the digitizer's initial state)
    int64_t global_offset;
    int64_t* row_off;
    int64_t* prev_fired;
    __device__ __forceinline__ FireAgg load(int64_t t) const {
        const TileFire f = fire[t];
        int prev = prev_cls[t];
        if (prev == CLS_NONE) prev = *d_prev0;
        FireAgg r;
        r.fired = f.fired;
        int32_t last = f.last_rel;
        if (f.first_cls != CLS_NONE && f.first_cls != prev) {
            r.fired++;
            if (last < 0) last = f.first_rel;
        }
        r.last_pos = (last >= 0) ? t * URH_TILE + global_offset + last : -1;
        return r;
    }
    __device__ __forceinline__ void post(int64_t t, const FireAgg& excl, const FireAgg&) const {
        row_off[t] = excl.fired;
        prev_fired[t] = excl.last_pos;
    }
};

// ---- the walk of stage D: one warp per run of FIN_TILES consecutive tiles ------------------------------------------------------
// A candidate fires iff its class differs from the one before it.  The lanes take a tile's staged words 32 at a time (one coalesced
// load from the tile's staging row), the predecessor's class with a shuffle (lane 0: the carried one), the firings with a ballot.
constexpr int FIN_TILES = 32;   // tiles per warp: lane i loads the per-tile scalars of the warp's i-th tile
constexpr int FIN_BATCH = 8;    // tiles whose first 32 staged words are loaded before the first of them is walked

struct FinRows {   // stage D's output
    int64_t* out;
    int64_t cap_rows;
    int tol;
    int is_ask;
    int64_t sps;
};

// What a tile's walk carries from one candidate to the next (warp-uniform).
struct FinWalk {
    int prev;         // class of the preceding candidate
    int64_t pp;       // position of the preceding firing (-1: none)
    int64_t idx;      // row of the next firing
};

// One firing, written by one lane: (state, length) at row idx (pyx:471-482); rows beyond cap_rows are dropped but counted.
__device__ __forceinline__ void fin_row(const FinRows& R, int64_t idx, int64_t p, int64_t pp, int prev) {
    // pulse lengths (pyx:476-482): the first pulse of the capture is counted from its start
    const int64_t rec = (pp >= 0) ? (p - pp) : (p + 1 - R.tol);
    int64_t st = prev;
    if (R.is_ask && st == -1 && rec < R.sps) st = 0;   // ASK: a pause shorter than one symbol is a zero (pyx:471-473)
    if (idx < R.cap_rows) *((longlong2*)R.out + idx) = make_longlong2(st, rec);   // one 16-byte store per row
}

// Up to 32 staged candidates of one tile: this lane's word w (lanes >= cnt: none).  Firing lanes write consecutive rows.
__device__ __forceinline__ void fin_chunk(FinWalk& W, uint32_t w, int cnt, int lane, int64_t base, const FinRows& R) {
    const int c = (int)(w & 0xffffu) - 1;
    const int rel = (int)(w >> 16);
    int pc = __shfl_up_sync(URH_FULL_MASK, c, 1);
    if (lane == 0) pc = W.prev;
    const bool fire = lane < cnt && c != pc;
    const unsigned fm = __ballot_sync(URH_FULL_MASK, fire);
    // the firing before this lane's: the highest firing lane below it (positions grow with the lane), else the carried one
    const unsigned lower = fm & ((1u << lane) - 1u);
    const int before = __shfl_sync(URH_FULL_MASK, rel, lower ? 31 - __clz(lower) : 0);
    if (fire) fin_row(R, W.idx + __popc(lower), base + rel, lower ? base + before : W.pp, pc);
    if (fm) W.pp = base + __shfl_sync(URH_FULL_MASK, rel, 31 - __clz(fm));
    W.idx += __popc(fm);
    if (cnt > 0) W.prev = __shfl_sync(URH_FULL_MASK, c, cnt - 1);
}

// ---- D ---------------------------------------------------------------------------------------------------------------
// out = (state, length) pairs; rows beyond cap_rows are dropped (the caller grows the buffer and repeats).
// d_out[0] = rows written incl. tail, d_out[1] = firings.  The warp's tiles [t0, t0 + FIN_TILES) in order: head candidate, then the
// staged ones.
__global__ void __launch_bounds__(256) k_finish_rows(const UrhTileSummary* __restrict__ tiles, const uint32_t* __restrict__ staging,
                                                    int stage_cap, const int32_t* __restrict__ head_rel, const int32_t* __restrict__ prev_cls,
                                                    const int16_t* __restrict__ d_prev0, const int64_t* __restrict__ row_off,
                                                    const int64_t* __restrict__ prev_fired, const int64_t* __restrict__ d_xprev_fired,
                                                    int64_t ntiles, int64_t global_offset, int64_t n_total, int tol, int is_ask, int64_t sps,
                                                    int emit_tail, int64_t row_base, int64_t* __restrict__ out, int64_t cap_rows,
                                                    int64_t* __restrict__ d_out) {
    const int64_t t0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32 * FIN_TILES;
    if (t0 >= ntiles) return;
    const int lane = threadIdx.x & 31;
    FinRows R;
    R.out = out; R.cap_rows = cap_rows; R.tol = tol; R.is_ask = is_ask; R.sps = sps;
    // lane i: the scalars of tile t0 + i
    const int64_t tl = t0 + lane;
    int l_first = 0, l_ncand = 0, l_rel = -1, l_prev = 0;
    int64_t l_idx = 0, l_pp = -1;
    if (tl < ntiles) {
        const UrhTileSummary s = tiles[tl];
        l_first = s.first_cls;
        l_ncand = s.ncand;
        l_rel = head_rel[tl];
        l_prev = prev_cls[tl];
        if (l_prev == CLS_NONE) l_prev = *d_prev0;
        l_idx = row_off[tl];
        l_pp = prev_fired[tl];
        if (l_pp < 0) l_pp = *d_xprev_fired;
    }
    for (int j0 = 0; j0 < FIN_TILES && t0 + j0 < ntiles; j0 += FIN_BATCH) {
        uint32_t w0[FIN_BATCH];
#pragma unroll
        for (int u = 0; u < FIN_BATCH; u++) {
            const int nc = __shfl_sync(URH_FULL_MASK, l_ncand, j0 + u);
            w0[u] = (lane < nc) ? __ldg(staging + (t0 + j0 + u) * (int64_t)stage_cap + lane) : 0u;
        }
#pragma unroll
        for (int u = 0; u < FIN_BATCH; u++) {
            const int j = j0 + u;
            const int64_t t = t0 + j;
            if (t >= ntiles) break;
            const int64_t base = t * URH_TILE + global_offset;
            const int ncand = __shfl_sync(URH_FULL_MASK, l_ncand, j);
            const int rel = __shfl_sync(URH_FULL_MASK, l_rel, j);
            FinWalk W;
            W.prev = __shfl_sync(URH_FULL_MASK, l_prev, j);
            W.pp = __shfl_sync(URH_FULL_MASK, l_pp, j);
            W.idx = __shfl_sync(URH_FULL_MASK, l_idx, j);
            if (rel >= 0) {   // the head candidate (a run entering the tile reaches the tolerance inside it)
                const int c = __shfl_sync(URH_FULL_MASK, l_first, j);
                if (c != W.prev) {
                    if (lane == 0) fin_row(R, W.idx, base + rel, W.pp, W.prev);
                    W.idx++;
                    W.pp = base + rel;
                }
                W.prev = c;
            }
            const uint32_t* st = staging + t * (int64_t)stage_cap;
            for (int k = 0; k < ncand; k += 32) {   // a tile holds up to stage_cap (1026 at tolerance 0) candidates
                const uint32_t w = (k == 0) ? w0[u] : ((k + lane < ncand) ? __ldg(st + k + lane) : 0u);
                fin_chunk(W, w, min(32, ncand - k), lane, base, R);
            }
            if (t == ntiles - 1 && lane == 0) {
                int64_t idx = W.idx;
                const int64_t fired = idx;
                // tail row (pyx:485-493): appended only while fewer than n rows exist (row_base: rows of the chunks before this one)
                if (emit_tail && (is_ask || row_base + fired < n_total)) {
                    if (idx < cap_rows) *((longlong2*)out + idx) = make_longlong2(W.prev, (W.pp >= 0) ? (n_total - 1 - W.pp) : (n_total - tol));
                    idx++;
                }
                d_out[0] = idx;
                d_out[1] = fired;
            }
        }
    }
}

// ---- ASK: merge equal neighbours (pyx:475-476) -------------------------------------------------------------------------
// A chained chunk (prev_last != nullptr) writes at out = table + row_base rows; a first row whose state equals the table's last
// row (*prev_last) is a head of 0 and lands at out[-1], i.e. it is added to that row, as merge_shard_rows joins shard edges.
struct ScanMergeRows {
    const int64_t* raw;    // (state, length) x rows, the tail row last when has_tail
    int64_t rows;
    int64_t n_total;
    int has_tail;
    int64_t* out;
    int64_t* d_k;
    const int64_t* prev_last;   // state of the row before out[0] (nullptr: none)
    int64_t row_base;           // rows before out[0]
    __device__ __forceinline__ int64_t load(int64_t r) const {
        if (r == 0) return (prev_last && raw[0] == *prev_last) ? 0 : 1;
        return raw[2 * r] != raw[2 * r - 2] ? 1 : 0;
    }
    __device__ __forceinline__ void post(int64_t r, const int64_t& excl, const int64_t& head) const {
        const bool is_tail = has_tail && r == rows - 1;
        // the tail row is appended only while fewer than n (merged) rows exist (pyx:487)
        if (is_tail && row_base + excl >= n_total) {
            *d_k = excl;
            return;
        }
        const int64_t o = excl + head - 1;
        if (head) out[2 * o] = raw[2 * r];
        atomicAdd((unsigned long long*)&out[2 * o + 1], (unsigned long long)raw[2 * r + 1]);
        if (r == rows - 1) *d_k = o + 1;
    }
};
struct AddI64 {
    __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};

// ---- folding the totals of the preceding ranks (sharded captures) ------------------------------------------------------------
// Stage-1 message of a rank: {RunCarry total (2 x int64), init class, pad}; stages 2 and 3: the CandAgg / FireAgg total.
__global__ void k_pack_stage1(const int16_t* __restrict__ d_init, const RunCarry* __restrict__ total, int64_t* __restrict__ msg) {
    memcpy(msg, total, sizeof(RunCarry));
    msg[2] = *d_init;
    msg[3] = 0;
}
__global__ void k_fold_carry(const int64_t* __restrict__ all, int rank, RunCarry* __restrict__ xcarry) {
    RunCarry acc;
    acc.len = 0; acc.cls = 0; acc.flags = 2 | 1;
    for (int q = 0; q < rank; q++) {
        RunCarry c;
        memcpy(&c, all + 4 * q, sizeof(c));
        acc = RunCarryOp()(acc, c);
    }
    if (rank == 0) acc.flags = 2;   // nothing precedes the first shard
    else acc.flags &= ~1;           // the incoming run is never "the whole span" of this shard
    *xcarry = acc;
}
__global__ void k_fold_prev_cls(const int64_t* __restrict__ all, int rank, const int64_t* __restrict__ stage1, int16_t* __restrict__ prev0) {
    int v = (int)stage1[2];   // rank 0's initial class
    for (int q = 0; q < rank; q++) {
        CandAgg c;
        memcpy(&c, all + 2 * q, sizeof(c));
        if (c.last_cls != CLS_NONE) v = c.last_cls;
    }
    *prev0 = (int16_t)v;
}
__global__ void k_fold_prev_fired(const int64_t* __restrict__ all, int rank, int64_t* __restrict__ xprev) {
    int64_t v = -1;
    for (int q = 0; q < rank; q++) {
        FireAgg c;
        memcpy(&c, all + 2 * q, sizeof(c));
        if (c.last_pos >= 0) v = c.last_pos;
    }
    *xprev = v;
}

// ---- chained chunks (streaming) -------------------------------------------------------------------------------------------------
// Before chunk 0's finish: the digitizer's initial state becomes the "previous class"; nothing precedes the capture.
__global__ void k_chain_start(const int16_t* __restrict__ d_init, UrhChain* __restrict__ chain) {
    chain->run.len = 0; chain->run.cls = 0; chain->run.flags = 2 | 1;
    chain->prev_fired = -1;
    chain->last_state = INT64_MIN;
    chain->prev_cls = *d_init;
}
// After a chunk's rows: fold its three scan totals into the chain, as k_fold_* fold the totals of the preceding ranks.
__global__ void k_chain_advance(UrhChain* __restrict__ chain, const RunCarry* __restrict__ tot_run, const CandAgg* __restrict__ tot_cand,
                                const FireAgg* __restrict__ tot_fire) {
    chain->run = RunCarryOp()(chain->run, *tot_run);
    if (tot_cand->last_cls != CLS_NONE) chain->prev_cls = (int16_t)tot_cand->last_cls;
    if (tot_fire->last_pos >= 0) chain->prev_fired = tot_fire->last_pos;
}
__global__ void k_chain_last_row(UrhChain* __restrict__ chain, const int64_t* __restrict__ table, int64_t rows) {
    if (rows > 0) chain->last_state = table[2 * (rows - 1)];
}

// ---- driver --------------------------------------------------------------------------------------------------------------
// A shard folds the three scan totals of the preceding ranks, exchanged on the stream; a chained chunk takes them from and folds
// them into *chain (device memory).
int finish_tiles(urh_ctx* ctx, const UrhDigitizer& dz, const FinishShard& sh, int64_t* k) {
    const int64_t n = sh.n;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const bool sharded = sh.world > 1;
    UrhChain* chain = sh.chain;
    RunCarry* carry;
    int32_t *head_rel, *prev_cls;
    int64_t *row_off, *prev_fired, *d_small;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &carry));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &head_rel));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &prev_cls));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &row_off));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &prev_fired));
    TileFire* fire;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &fire));
    // small block (int64 units): [0..1] stage D's outputs, [2] -1 (no previous firing), [4..5] RunCarry total, [6..7] CandAgg total,
    // [8..9] FireAgg total, [10..11] folded run carry, [12] folded previous class (int16), [13] folded previous firing,
    // [16..19] stage-1 message, [32..) gathered messages: world x 4 (stage 1), world x 2 (stage 2), world x 2 (stage 3)
    URH_CHECK(urh_arena(ctx, (size_t)(32 + 8 * (sharded ? sh.world : 0)), &d_small));
    URH_CUDA(ctx, cudaMemsetAsync(d_small, 0xff, 4 * sizeof(int64_t), ctx->stream));
    RunCarry* d_tot_run = (RunCarry*)(d_small + 4);
    CandAgg* d_tot_cand = (CandAgg*)(d_small + 6);
    FireAgg* d_tot_fire = (FireAgg*)(d_small + 8);
    RunCarry* d_xcarry = (RunCarry*)(d_small + 10);
    int16_t* d_prev0 = (int16_t*)(d_small + 12);
    int64_t* d_xprev = d_small + 13;
    int64_t* d_msg1 = d_small + 16;
    int64_t* d_all1 = d_small + 32;
    int64_t* d_all2 = d_all1 + 4 * (sharded ? sh.world : 0);
    int64_t* d_all3 = d_all2 + 2 * (sharded ? sh.world : 0);

    if (chain && sh.global_offset == 0) URH_LAUNCH(ctx, k_chain_start, 1, 1, 0, dz.d_init, chain);
    RunCarry rc_ident;
    rc_ident.len = 0; rc_ident.cls = 0; rc_ident.flags = 2 | 1;
    ScanRunCarry fa;
    fa.tiles = dz.tiles; fa.n = n; fa.carry = carry;
    URH_CHECK((urhts::scan<RunCarry, RunCarryOp, ScanRunCarry>(ctx, ntiles, rc_ident, RunCarryOp(), fa, d_tot_run)));
    if (sharded) {
        URH_LAUNCH(ctx, k_pack_stage1, 1, 1, 0, dz.d_init, (const RunCarry*)d_tot_run, d_msg1);
        URH_TL_MARK(ctx, "x4 run carry: enter");
        URH_CHECK(urh_nccl_allgather(ctx, d_msg1, d_all1, 4 * sizeof(int64_t)));
        URH_TL_MARK(ctx, "x4 run carry: done");
        URH_LAUNCH(ctx, k_fold_carry, 1, 1, 0, (const int64_t*)d_all1, sh.rank, d_xcarry);
    }
    ScanCandidates fb;
    fb.tiles = dz.tiles; fb.staging = dz.staging; fb.stage_cap = dz.cap; fb.carry = carry;
    fb.xcarry = sharded ? d_xcarry : (chain ? &chain->run : nullptr);
    fb.tol = dz.tol; fb.head_rel = head_rel; fb.prev_cls = prev_cls; fb.fire = fire;
    CandAgg ca_ident;
    ca_ident.cnt = 0; ca_ident.last_cls = CLS_NONE; ca_ident.pad = 0;
    URH_CHECK((urhts::scan<CandAgg, CandOp, ScanCandidates, 4>(ctx, ntiles, ca_ident, CandOp(), fb, d_tot_cand)));   // heavy load(): thin blocks
    const int16_t* prev0 = chain ? &chain->prev_cls : dz.d_init;
    if (sharded) {
        URH_TL_MARK(ctx, "x5 candidates: enter");
        URH_CHECK(urh_nccl_allgather(ctx, d_tot_cand, d_all2, sizeof(CandAgg)));
        URH_TL_MARK(ctx, "x5 candidates: done");
        URH_LAUNCH(ctx, k_fold_prev_cls, 1, 1, 0, (const int64_t*)d_all2, sh.rank, (const int64_t*)d_all1, d_prev0);
        prev0 = d_prev0;
    }
    ScanFirings fc;
    fc.fire = fire; fc.prev_cls = prev_cls; fc.d_prev0 = prev0; fc.global_offset = sh.global_offset; fc.row_off = row_off;
    fc.prev_fired = prev_fired;
    FireAgg fi_ident;
    fi_ident.fired = 0; fi_ident.last_pos = -1;
    URH_CHECK((urhts::scan<FireAgg, FireOp, ScanFirings>(ctx, ntiles, fi_ident, FireOp(), fc, d_tot_fire)));
    const int64_t* xprev = chain ? &chain->prev_fired : d_small + 2;
    if (sharded) {
        URH_TL_MARK(ctx, "x6 firings: enter");
        URH_CHECK(urh_nccl_allgather(ctx, d_tot_fire, d_all3, sizeof(FireAgg)));
        URH_TL_MARK(ctx, "x6 firings: done");
        URH_LAUNCH(ctx, k_fold_prev_fired, 1, 1, 0, (const int64_t*)d_all3, sh.rank, d_xprev);
        xprev = d_xprev;
    }

    // rows: straight into the pulse buffer (ASK: into scratch, merged afterwards)
    int64_t cap_rows = (int64_t)ctx->pulses_cap_rows;
    const int64_t guess = n / 64 + 1024;
    if (!chain && cap_rows < guess) {
        URH_CHECK(urh_ensure_pulses(ctx, (size_t)guess));
        cap_rows = (int64_t)ctx->pulses_cap_rows;
    }
    const int64_t row_base = chain ? sh.row_base : 0;
    int64_t* raw = ctx->pulses + 2 * row_base;
    int64_t raw_cap = chain ? sh.rows_cap : cap_rows;
    if (dz.is_ask) URH_CHECK(urh_arena(ctx, (size_t)raw_cap * 2, &raw));
    int64_t got[2] = {0, 0};
    for (int attempt = 0; attempt < 2; attempt++) {
        URH_LAUNCH(ctx, k_finish_rows, (unsigned)urh_div_up(ntiles, 8 * FIN_TILES), 256, 0, dz.tiles, dz.staging, dz.cap, (const int32_t*)head_rel,
                   (const int32_t*)prev_cls, prev0, (const int64_t*)row_off, (const int64_t*)prev_fired, xprev, ntiles, sh.global_offset,
                   sh.n_total, dz.tol, dz.is_ask ? 1 : 0, (int64_t)dz.sps, sh.emit_tail, row_base, raw, raw_cap, d_small);
        if (sharded && attempt == 0) URH_TL_MARK(ctx, "rows written");
        URH_CHECK(urh_read_i64(ctx, d_small, 2, got));
        if (got[0] <= raw_cap) break;
        // rows_cap bounds a chained chunk's rows (one per candidate plus the tail), so only the unchained table can overflow
        if (attempt == 1 || chain) URH_FAIL(ctx, URH_ERR_CUDA, "finish_tiles: row buffer overflow after regrowth");
        // more rows than guessed: grow and repeat stage D only
        if (dz.is_ask) {
            URH_CHECK(urh_arena(ctx, (size_t)got[0] * 2, &raw));
            raw_cap = got[0];
        } else {
            URH_CHECK(urh_ensure_pulses(ctx, (size_t)got[0]));
            raw = ctx->pulses;
            raw_cap = (int64_t)ctx->pulses_cap_rows;
        }
    }
    if (chain) URH_LAUNCH(ctx, k_chain_advance, 1, 1, 0, chain, (const RunCarry*)d_tot_run, (const CandAgg*)d_tot_cand, (const FireAgg*)d_tot_fire);
    int64_t K = got[0];
    if (dz.is_ask && K > 0) {
        if (!chain) URH_CHECK(urh_ensure_pulses(ctx, (size_t)K));
        int64_t* out = ctx->pulses + 2 * row_base;
        URH_CUDA(ctx, cudaMemsetAsync(out, 0, (size_t)K * 2 * sizeof(int64_t), ctx->stream));
        ScanMergeRows fm;
        fm.raw = raw; fm.rows = K; fm.n_total = sh.n_total; fm.has_tail = (sh.emit_tail && K > got[1]) ? 1 : 0; fm.out = out;
        fm.d_k = d_small;
        fm.prev_last = (chain && row_base > 0) ? &chain->last_state : nullptr;
        fm.row_base = row_base;
        URH_CHECK((urhts::scan<int64_t, AddI64, ScanMergeRows>(ctx, K, (int64_t)0, AddI64(), fm, (int64_t*)nullptr)));
        URH_CHECK(urh_read_i64(ctx, d_small, 1, &K));
        if (chain) URH_LAUNCH(ctx, k_chain_last_row, 1, 1, 0, chain, (const int64_t*)ctx->pulses, row_base + K);
    }
    ctx->pulses_k = row_base + K;
    *k = K;
    return URH_OK;
}
