// Sparse stages shared by the digitizer, the message segmenter and the plateau RLE:
// tile summaries + per-tile staged candidates  ->  one ordered, compact candidate table.
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

// grab_pulse_lens tail (signal_functions.pyx:455-495) on the candidate table: fire filter, pulse lengths,
// ASK short-pause relabel, merge of equal neighbours, tail row.  Result -> ctx->pulses / ctx->pulses_k.
int urh_pulses_from_candidates(urh_ctx* ctx, int64_t n, int tol, bool is_ask, uint32_t sps, const UrhCandidates& cand,
                               const int16_t* d_init_cls, int64_t* k);

// The two halves of urh_pulses_from_candidates, separable so that shards can exchange the two scalars each half
// needs from its predecessors: the class of the last candidate before the shard (fire decision of its first
// candidate) and the position of the last firing before the shard (length of its first pulse).
struct UrhFireState {
    int64_t C, F;
    int64_t* fire;
    const int64_t* pos;
    const int16_t* cls;
    const int16_t* d_prev_cls;
    int64_t *fpos, *st, *ln, *head;
};
int urh_fire_stage(urh_ctx* ctx, const UrhCandidates& cand, const int16_t* d_prev_cls, UrhFireState* fs, int64_t* last_fired_pos);
int urh_rows_stage(urh_ctx* ctx, const UrhFireState& fs, int64_t n, int tol, bool is_ask, uint32_t sps, int64_t prev_fired,
                   bool emit_tail, int64_t* k);
