// Run stitching across tiles (RunCarry), used by the digitizer's tile-level finish (finish.cu), and the gathered candidate table of
// the message segmenter and the plateau RLE (stats.cu): tile summaries + per-tile staged candidates  ->  one ordered, compact table.
// UrhChain: what a chunk's finish receives from the chunks before it; UrhDigitizer and FinishShard: what a finish reads and where
// its rows go (finish.cu).
#pragma once
#include "dense.cuh"

// The run that ends at the end of a span of tiles, and the associative operator that concatenates two spans.
struct __align__(16) RunCarry {
    int64_t len;    // length of the run that ends at the end of the span
    int32_t cls;    // its class
    int32_t flags;  // bit0: the whole span is one run; bit1: empty span (identity)
};
struct RunCarryOp {
    __device__ __forceinline__ RunCarry operator()(const RunCarry& a, const RunCarry& b) const {
        if (b.flags & 2) return a;
        if (a.flags & 2) return b;
        RunCarry r;
        if ((b.flags & 1) && b.cls == a.cls) {
            r.len = a.len + b.len;
            r.cls = a.cls;
            r.flags = a.flags & 1;
        } else {
            r.len = b.len;
            r.cls = b.cls;
            r.flags = 0;
        }
        return r;
    }
};

// The look-back scan's element (tilescan.cuh) for run stitching over a tile table of n samples: tile t's closing run, whole if
// the tile is one run.  Callers add the post hook that consumes the carries.
struct TileRuns {
    const UrhTileSummary* tiles;
    int64_t n;
    __device__ __forceinline__ RunCarry load(int64_t t) const {
        const int64_t rem = n - t * URH_TILE;
        const int tile_len = rem < URH_TILE ? (int)rem : URH_TILE;
        const UrhTileSummary s = tiles[t];
        RunCarry r;
        r.len = s.tail_len;
        r.cls = s.last_cls;
        r.flags = (s.head_len == tile_len) ? 1 : 0;
        return r;
    }
};

// Chunks of one capture digitized one after another on the same GPU (streaming, finish.cu): what the finish of chunk c needs from
// the chunks before it, left in device memory by their finishes.  The same three totals a shard receives from its predecessors.
struct __align__(16) UrhChain {
    RunCarry run;          // the run that ends at the end of the preceding chunks (identity before chunk 0)
    int64_t prev_fired;    // position of the last firing in the preceding chunks (-1: none)
    int64_t last_state;    // state of the last row in the pulse table (ASK merge across the chunk edge)
    int16_t prev_cls;      // class of the last candidate of the preceding chunks (chunk 0: the digitizer's initial state)
    int16_t pad[7];
};

// staged candidates per tile of a digitizer at tolerance tol: firings are >= tol + 1 samples apart
static inline int stage_cap_for(int tol) { return URH_TILE / (tol + 1) + 2; }

// The digitizer of one pulse table: the dense pass fills the tile summaries, the staged candidates of each tile and the initial
// state; finish_tiles turns them into (state, length) rows.
struct UrhDigitizer {
    int64_t n;                // samples the pulse table covers (a shard: its own)
    int tol, cap;             // tolerance; staged candidates per tile
    bool is_ask;
    uint32_t sps;             // samples per symbol
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;          // the initial state, stored by the pass over the capture's first tile
    // The tables for ntiles tiles from the arena.  zero_init: d_init is zeroed now, on the stream.
    int init(urh_ctx* ctx, int64_t n_, int tol_, bool ask, uint32_t sps_, int64_t ntiles, bool zero_init) {
        n = n_; tol = tol_; cap = stage_cap_for(tol); is_ask = ask; sps = sps_;
        URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
        URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
        URH_CHECK(urh_arena(ctx, 8, &d_init));
        if (zero_init) URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
        return URH_OK;
    }
};

// Which rows a finish writes and what precedes them: the whole capture, one shard of the context's NCCL communicator, or a chunk
// of a capture streamed through this GPU.
struct FinishShard {
    int64_t n;                  // samples of this shard (chunk)
    int rank, world;            // world == 1: unsharded
    int64_t global_offset;      // first sample of this shard in the capture
    int64_t n_total;
    int emit_tail;
    // chained chunk: the carries come from *chain instead of the other ranks, and the rows are appended to the pulse table after
    // its first row_base rows (the caller has made room for rows_cap more)
    UrhChain* chain;
    int64_t row_base, rows_cap;

    static FinishShard local(const UrhDigitizer& dz) { return FinishShard{dz.n, 0, 1, 0, dz.n, 1, nullptr, 0, 0}; }
    // every rank ends with the rows of its own shard; equal states meeting at a shard edge are joined by the consumer
    static FinishShard shard(const urh_ctx* ctx, const UrhDigitizer& dz, int64_t global_offset, int64_t n_total) {
        return FinishShard{dz.n, ctx->nccl_rank, ctx->nccl_world, global_offset, n_total, ctx->nccl_rank == ctx->nccl_world - 1 ? 1 : 0,
                           nullptr, 0, 0};
    }
    // the chunk [s0, s1) of a capture of n_total samples; a first row that continues the table's last row is merged into it
    static FinishShard chunk(UrhChain* chain, int64_t s0, int64_t s1, int64_t n_total, int64_t row_base, int64_t rows_cap) {
        return FinishShard{s1 - s0, 0, 1, s0, n_total, s1 == n_total ? 1 : 0, chain, row_base, rows_cap};
    }
};
// The pulse table of the tiles dz's dense pass filled (finish.cu).  *k = the rows this finish added.
int finish_tiles(urh_ctx* ctx, const UrhDigitizer& dz, const FinishShard& sh, int64_t* k);

// The tile table of a dense pass with a binary classifier over n samples (the segmenter, the plateau RLE; stats.cu)
struct UrhRunTable {
    int64_t n;
    int tol, cap;             // tolerance; staged candidates per tile
    UrhTileSummary* tiles;
    uint32_t* staging;
};

struct UrhCandidates {
    int64_t count;   // number of candidates (host copy)
    int64_t* pos;    // device: absolute sample index run_start + tolerance
    int16_t* cls;    // device: class of the run
    // the run that contains the LAST sample of the table, without the carry (host copies): class, length, 1 if it is the whole table
    int32_t last_cls;
    int64_t last_len;
    int whole;
};

// The run that ends at the end of the PRECEDING shards or chunks (class, length); valid = 0 for the first one.
struct UrhShardCarry {
    int valid;
    int cls;
    int64_t len;
};
// Stitch runs across tile edges (scan over the tile table) from the carry, add the per-tile head candidates and gather everything
// into `out` (arena memory), positions offset by `global_offset` (the table's first sample index in the whole capture).
// Synchronises once to learn the candidate count.
int urh_collect_candidates_shard(urh_ctx* ctx, const UrhRunTable& rt, UrhShardCarry carry_in, int64_t global_offset, UrhCandidates* out);
// The shard's own run summary for the exchange before its candidates are collected: h_out = {last_cls, last_len, whole (1 if the
// shard is one run)}.
int urh_shard_run_total(urh_ctx* ctx, int64_t n, const UrhTileSummary* tiles, int64_t* h_out);

