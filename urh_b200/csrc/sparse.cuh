// Run stitching across tiles (RunCarry), used by the digitizer's tile-level finish (finish.cu), and the gathered candidate table of
// the message segmenter and the plateau RLE (stats.cu): tile summaries + per-tile staged candidates  ->  one ordered, compact table.
// UrhChain: what a chunk's finish receives from the chunks before it (finish.cu).
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

struct UrhCandidates {
    int64_t count;   // number of candidates (host copy)
    int64_t* pos;    // device: absolute sample index run_start + tolerance
    int16_t* cls;    // device: class of the run
    // the run that contains the LAST sample of the stream (host copies): class and length
    int32_t last_cls;
    int64_t last_len;
};

// Stitch runs across tile edges (scan over the tile table), add the per-tile head candidates and gather
// everything into `out` (arena memory).  Synchronises once to learn the candidate count.
int urh_collect_candidates(urh_ctx* ctx, int64_t n, int tol, const UrhTileSummary* tiles, const uint32_t* staging,
                           int stage_cap, UrhCandidates* out);

// Sharded captures: the run that ends at the end of the PRECEDING shards (class, length); valid = 0 for the first shard.
struct UrhShardCarry {
    int valid;
    int cls;
    int64_t len;
};
// As urh_collect_candidates, with the carry of the preceding shards folded in and positions offset by
// `global_offset` (the shard's first sample index in the whole capture).
int urh_collect_candidates_shard(urh_ctx* ctx, int64_t n, int tol, const UrhTileSummary* tiles, const uint32_t* staging,
                                 int stage_cap, UrhShardCarry carry_in, int64_t global_offset, UrhCandidates* out);
// The shard's own run summary for the exchange: h_out = {last_cls, last_len, whole (1 if the shard is one run)}.
int urh_shard_run_total(urh_ctx* ctx, int64_t n, const UrhTileSummary* tiles, int64_t* h_out);

