// Run stitching and candidate collection over a tile table: the segmenter's and the plateau RLE's candidate tables and a shard's
// closing run (see sparse.cuh, DESIGN.md §4.2).
#include "sparse.cuh"
#include "tilescan.cuh"

// ---- run stitching across tiles (RunCarry / RunCarryOp / TileRuns: sparse.cuh) -----------------------------------
// only the total: the run that ends the table
struct RunTotal : TileRuns {
    __device__ __forceinline__ void post(int64_t, const RunCarry&, const RunCarry&) const {}
};

// head candidate of each tile from the carry of all preceding tiles (and of the preceding shards, if any)
struct RunHeads : TileRuns {
    int tol;
    int has_in;
    RunCarry in;
    int32_t* head_rel;
    __device__ __forceinline__ void post(int64_t t, const RunCarry& excl, const RunCarry&) const {
        const RunCarry c = has_in ? RunCarryOp()(in, excl) : excl;
        const UrhTileSummary s = tiles[t];
        int64_t start_len = 0;
        if (!(c.flags & 2) && c.cls == s.first_cls) start_len = c.len;
        int32_t rel = -1;
        if (start_len <= tol && (int64_t)tol < start_len + s.head_len) rel = (int32_t)(tol - start_len);
        head_rel[t] = rel;
    }
};

// candidates of each tile (its head candidate and the staged ones) -> offset of the tile's first candidate in the table
struct CandOffsets {
    const UrhTileSummary* tiles;
    const int32_t* head_rel;
    int64_t* offset;
    __device__ __forceinline__ int64_t load(int64_t t) const { return (int64_t)tiles[t].ncand + (head_rel[t] >= 0 ? 1 : 0); }
    __device__ __forceinline__ void post(int64_t t, const int64_t& excl, const int64_t&) const { offset[t] = excl; }
};

static RunCarry run_identity() {
    RunCarry ident;
    ident.len = 0;
    ident.cls = 0;
    ident.flags = 2 | 1;
    return ident;
}

// one warp per tile: head candidate first, then the staged interior candidates
__global__ void k_gather(const UrhTileSummary* __restrict__ tiles, const uint32_t* __restrict__ staging, int stage_cap,
                         const int32_t* __restrict__ head_rel, const int64_t* __restrict__ offset, int64_t ntiles,
                         int64_t global_offset, int64_t* __restrict__ pos, int16_t* __restrict__ cls) {
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= ntiles) return;
    const UrhTileSummary s = tiles[t];
    int64_t o = offset[t];
    const int64_t base = t * URH_TILE + global_offset;
    const int32_t rel = head_rel[t];
    if (rel >= 0) {
        if (lane == 0) {
            pos[o] = base + rel;
            cls[o] = s.first_cls;
        }
        o++;
    }
    const uint32_t* st = staging + t * (int64_t)stage_cap;
    for (int j = lane; j < s.ncand; j += 32) {
        const uint32_t v = st[j];
        pos[o + j] = base + (v >> 16);
        cls[o + j] = (int16_t)((int)(v & 0xffff) - 1);
    }
}

int urh_shard_run_total(urh_ctx* ctx, int64_t n, const UrhTileSummary* tiles, int64_t* h_out) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    RunCarry* d_total_run;
    URH_CHECK(urh_arena(ctx, 2, &d_total_run));
    RunTotal f;
    f.tiles = tiles; f.n = n;
    URH_CHECK((urhts::scan<RunCarry, RunCarryOp, RunTotal>(ctx, ntiles, run_identity(), RunCarryOp(), f, d_total_run)));
    int64_t raw[2];
    URH_CHECK(urh_read_i64(ctx, (const int64_t*)d_total_run, 2, raw));
    RunCarry tr;
    memcpy(&tr, raw, sizeof(tr));
    h_out[0] = tr.cls;
    h_out[1] = tr.len;
    h_out[2] = (tr.flags & 1) ? 1 : 0;
    return URH_OK;
}

int urh_collect_candidates_shard(urh_ctx* ctx, const UrhRunTable& rt, UrhShardCarry carry_in, int64_t global_offset, UrhCandidates* out) {
    const int64_t n = rt.n;
    const UrhTileSummary* tiles = rt.tiles;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    int32_t* head_rel;
    int64_t* offset;
    int64_t* d_count;
    RunCarry* d_total_run;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &head_rel));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &offset));
    URH_CHECK(urh_arena(ctx, 4, &d_count));
    URH_CHECK(urh_arena(ctx, 2, &d_total_run));
    RunHeads fh;
    fh.tiles = tiles; fh.n = n; fh.tol = rt.tol; fh.head_rel = head_rel;
    fh.has_in = carry_in.valid ? 1 : 0;
    fh.in.len = carry_in.len; fh.in.cls = carry_in.cls; fh.in.flags = 0;
    // the total is the shard's own closing run, without the carry of the preceding shards
    URH_CHECK((urhts::scan<RunCarry, RunCarryOp, RunHeads>(ctx, ntiles, run_identity(), RunCarryOp(), fh, d_total_run)));
    CandOffsets fc;
    fc.tiles = tiles; fc.head_rel = head_rel; fc.offset = offset;
    URH_CHECK((urhts::scan<int64_t, urhts::AddI64, CandOffsets>(ctx, ntiles, (int64_t)0, urhts::AddI64(), fc, d_count)));
    int64_t C = 0;
    URH_CHECK(urh_read_i64(ctx, d_count, 1, &C));
    {
        int64_t raw[2];
        URH_CHECK(urh_read_i64(ctx, (const int64_t*)d_total_run, 2, raw));
        RunCarry tr;
        memcpy(&tr, raw, sizeof(tr));
        out->last_cls = tr.cls;
        out->last_len = tr.len;
        out->whole = (tr.flags & 1) ? 1 : 0;
    }
    out->count = C;
    out->pos = nullptr;
    out->cls = nullptr;
    if (C == 0) return URH_OK;
    URH_CHECK(urh_arena(ctx, (size_t)C, &out->pos));
    URH_CHECK(urh_arena(ctx, (size_t)C, &out->cls));
    const unsigned gg = (unsigned)urh_div_up(ntiles * 32, 256);
    URH_LAUNCH(ctx, k_gather, gg, 256, 0, tiles, rt.staging, rt.cap, head_rel, offset, ntiles, global_offset, out->pos, out->cls);
    return URH_OK;
}
