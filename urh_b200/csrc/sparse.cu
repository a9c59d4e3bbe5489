// Run stitching and candidate collection over a tile table: the segmenter's and the plateau RLE's candidate tables and a shard's
// closing run (see sparse.cuh, DESIGN.md §4.2).
#include "sparse.cuh"
#include "scan.cuh"

// ---- run stitching across tiles (RunCarry / RunCarryOp: sparse.cuh) -------------------------------------
__global__ void k_tile_elems(const UrhTileSummary* __restrict__ tiles, int64_t ntiles, int64_t n, RunCarry* __restrict__ e) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    const int64_t rem = n - t * URH_TILE;
    const int tile_len = rem < URH_TILE ? (int)rem : URH_TILE;
    const UrhTileSummary s = tiles[t];
    RunCarry r;
    r.len = s.tail_len;
    r.cls = s.last_cls;
    r.flags = (s.head_len == tile_len) ? 1 : 0;
    e[t] = r;
}

// head candidate of each tile from the carry of all preceding tiles
__global__ void k_tile_heads(const UrhTileSummary* __restrict__ tiles, const RunCarry* __restrict__ carry,
                             int64_t ntiles, int tol, int32_t* __restrict__ head_rel, int64_t* __restrict__ total) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    const UrhTileSummary s = tiles[t];
    const RunCarry c = carry[t];
    int64_t start_len = 0;
    if (!(c.flags & 2) && c.cls == s.first_cls) start_len = c.len;
    int32_t rel = -1;
    if (start_len <= tol && (int64_t)tol < start_len + s.head_len) rel = (int32_t)(tol - start_len);
    head_rel[t] = rel;
    total[t] = (int64_t)s.ncand + (rel >= 0 ? 1 : 0);
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

__global__ void k_apply_carry(RunCarry* __restrict__ carry, int64_t ntiles, RunCarry in) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    carry[t] = RunCarryOp()(in, carry[t]);
}

int urh_shard_run_total(urh_ctx* ctx, int64_t n, const UrhTileSummary* tiles, int64_t* h_out) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    RunCarry* carry;
    RunCarry* d_total_run;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &carry));
    URH_CHECK(urh_arena(ctx, 2, &d_total_run));
    URH_LAUNCH(ctx, k_tile_elems, (unsigned)urh_div_up(ntiles, 256), 256, 0, tiles, ntiles, n, carry);
    RunCarry ident;
    ident.len = 0; ident.cls = 0; ident.flags = 2 | 1;
    URH_CHECK((urhscan::device_scan<RunCarry, RunCarryOp>(ctx, carry, ntiles, RunCarryOp(), ident, true, d_total_run)));
    int64_t raw[2];
    URH_CHECK(urh_read_i64(ctx, (const int64_t*)d_total_run, 2, raw));
    RunCarry tr;
    memcpy(&tr, raw, sizeof(tr));
    h_out[0] = tr.cls;
    h_out[1] = tr.len;
    h_out[2] = (tr.flags & 1) ? 1 : 0;
    return URH_OK;
}

int urh_collect_candidates(urh_ctx* ctx, int64_t n, int tol, const UrhTileSummary* tiles, const uint32_t* staging,
                           int stage_cap, UrhCandidates* out) {
    UrhShardCarry none;
    none.valid = 0; none.cls = 0; none.len = 0;
    return urh_collect_candidates_shard(ctx, n, tol, tiles, staging, stage_cap, none, 0, out);
}

int urh_collect_candidates_shard(urh_ctx* ctx, int64_t n, int tol, const UrhTileSummary* tiles, const uint32_t* staging,
                                 int stage_cap, UrhShardCarry carry_in, int64_t global_offset, UrhCandidates* out) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    RunCarry* carry;
    int32_t* head_rel;
    int64_t* total;
    int64_t* d_count;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &carry));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &head_rel));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &total));
    URH_CHECK(urh_arena(ctx, 4, &d_count));
    const unsigned g = (unsigned)urh_div_up(ntiles, 256);
    URH_LAUNCH(ctx, k_tile_elems, g, 256, 0, tiles, ntiles, n, carry);
    RunCarry ident;
    ident.len = 0;
    ident.cls = 0;
    ident.flags = 2 | 1;
    RunCarry* d_total_run;
    URH_CHECK(urh_arena(ctx, 2, &d_total_run));
    URH_CHECK((urhscan::device_scan<RunCarry, RunCarryOp>(ctx, carry, ntiles, RunCarryOp(), ident, true, d_total_run)));
    if (carry_in.valid) {
        RunCarry in;
        in.len = carry_in.len; in.cls = carry_in.cls; in.flags = 0;
        URH_LAUNCH(ctx, k_apply_carry, g, 256, 0, carry, ntiles, in);
    }
    URH_LAUNCH(ctx, k_tile_heads, g, 256, 0, tiles, carry, ntiles, tol, head_rel, total);
    URH_CHECK((urhscan::device_scan<int64_t, urhscan::AddI64>(ctx, total, ntiles, urhscan::AddI64(), (int64_t)0, true, d_count)));
    int64_t C = 0;
    URH_CHECK(urh_read_i64(ctx, d_count, 1, &C));
    {
        int64_t raw[2];
        URH_CHECK(urh_read_i64(ctx, (const int64_t*)d_total_run, 2, raw));
        RunCarry tr;
        memcpy(&tr, raw, sizeof(tr));
        out->last_cls = tr.cls;
        out->last_len = tr.len;
    }
    out->count = C;
    out->pos = nullptr;
    out->cls = nullptr;
    if (C == 0) return URH_OK;
    URH_CHECK(urh_arena(ctx, (size_t)C, &out->pos));
    URH_CHECK(urh_arena(ctx, (size_t)C, &out->cls));
    const unsigned gg = (unsigned)urh_div_up(ntiles * 32, 256);
    URH_LAUNCH(ctx, k_gather, gg, 256, 0, tiles, staging, stage_cap, head_rel, total, ntiles, global_offset, out->pos, out->cls);
    return URH_OK;
}
