// Shared internals of liburh_b200: context, error handling, scratch arena, launch accounting.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../include/urh_b200.h"

#define URH_FULL_MASK 0xffffffffu

struct urh_block {
    void* ptr;
    size_t bytes;
};

struct urh_ctx {
    int device;
    int sm_count;
    cudaStream_t stream;
    cudaStream_t copy_stream[2];
    cudaEvent_t ev_start, ev_stop;
    cudaEvent_t ev_copy[2], ev_comp[2];
    cudaEvent_t ev_k0, ev_k1;  // around the dense kernel when profiling is on
    int profiling;
    int dense_timed;
    // stream timeline (urh_set_profiling(ctx, 2)): events recorded at named points of the sharded step
    cudaEvent_t tl_ev[32];
    const char* tl_name[32];
    int tl_count, tl_ready;
    char err[512];
    int64_t launches;
    // grow-only scratch arena: bump allocation inside a list of blocks, reset at the start of each op
    std::vector<urh_block> arena;
    size_t arena_block;  // current block
    size_t arena_used;   // bytes used in current block
    size_t arena_need;   // bytes requested since last reset (for coalescing)
    // digitizer result (context-owned, separate from the arena so it survives the next op's reset)
    int64_t* pulses;
    size_t pulses_cap_rows;
    int64_t pulses_k;
    // small pinned host mailbox for scalar read-backs
    int64_t* h_mail;
    // pinned staging for the host-pointer entry points
    void* h_stage[2];
    size_t h_stage_bytes;
    // cuFFT plan cache (spectrogram.cu)
    int fft_plan;
    int fft_nfft;
    int64_t fft_batch;
    bool fft_valid;
    // twiddles of the last window size urh_spectrogram_bgra ran with (spectrogram.cu; 4096 entries allocated)
    void* img_tw;
    int img_tw_n;
    // sharded segmenter state between urh_segment_shard_pass and urh_shard_candidates / urh_fetch_candidates (stats.cu)
    void* shard_state;
    // NCCL (nccl.cu)
    int64_t costas_stats[3];
    int64_t costas_redone;  // super-chunks the stitch pass had to chain itself
    int64_t costas_stitch[4];  // {super-chunks adopted from family A, from family B, chained by the stitch warp, segs}
    void* costas_shard;   // the sharded PSK run between urh_costas_shard_speculate and its adopt / resolve (costas_spec.cu)
    // cuFFT plans of detect_modulation / cwt_haar: [0] C2C, [1] Z2Z, batch 2, length mod_plan_n
    int mod_plan[2];
    int mod_plan_valid[2];
    int64_t mod_plan_n[2];
    // urh_ppseq_to_bits results (arena)
    int bits_valid;
    int64_t bits_nmsg, bits_total, bits_npos;
    void *bits_ptr, *bits_msg_off, *bits_pauses, *bits_pos;
    const void* center_ts;
    const void* center_x;
    int64_t center_n;
    void* center_prefix;  // tile rank prefix left by urh_afp_demod_stats for urh_center_histogram_tiles (arena)
    int64_t center_cert[3];  // urh_center_certify_stats of the last one-call step
    int64_t spec_stats[3];   // urh_speculate_stats of the last one-call step
    void* nccl_comm;
    void* nccl_stage;
    void* nccl_hstage;  // pinned twin of nccl_stage
    int nccl_rank, nccl_world;
    // tilescan.cuh workspace (the look-back scans)
    void* ts_mem;
    int64_t ts_cap_blocks;
    unsigned long long ts_issued;
    uint32_t ts_epoch;
    // finish.cu / center chain: small device-resident result block and its pinned mirror
    void* step_dev;
    // digitizer exchange state of a sharded capture (finish.cu)
    void* shard_fin;
    // last streamed call (digitize.cu): lowest free device memory seen after a chunk, number of chunks
    int64_t stream_free_low, stream_chunks;
    size_t arena_live;   // bytes of the arena requests live since the last reset (released ones not counted)
    size_t arena_peak;   // the most arena_live reached since the last reset
    // (start, end) pairs of the last urh_segment_messages(_iq_stream) call (urh_fetch_segments)
    std::vector<int64_t> segments;
};

#define URH_CUDA(ctx, call)                                                                         \
    do {                                                                                            \
        cudaError_t e__ = (call);                                                                   \
        if (e__ != cudaSuccess) {                                                                   \
            snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,  \
                     cudaGetErrorString(e__));                                                      \
            return (e__ == cudaErrorMemoryAllocation) ? URH_ERR_NOMEM : URH_ERR_CUDA;               \
        }                                                                                           \
    } while (0)

#define URH_CHECK(call)                 \
    do {                                \
        int rc__ = (call);              \
        if (rc__ != URH_OK) return rc__; \
    } while (0)

#define URH_FAIL(ctx, code, ...)                                  \
    do {                                                          \
        snprintf((ctx)->err, sizeof((ctx)->err), __VA_ARGS__);    \
        return (code);                                            \
    } while (0)

// Kernel launch with accounting + error check.
#define URH_LAUNCH(ctx, kernel, grid, block, smem, ...)                                   \
    do {                                                                                  \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                  \
        (ctx)->launches++;                                                                \
        URH_CUDA(ctx, cudaGetLastError());                                                \
    } while (0)

// stream timeline: mark a point of the step (profiling level 2 only; no effect otherwise)
#define URH_TL_MARK(ctx, label) do { if ((ctx)->profiling >= 2 && (ctx)->tl_ready && (ctx)->tl_count < 32) { \
        (ctx)->tl_name[(ctx)->tl_count] = (label); cudaEventRecord((ctx)->tl_ev[(ctx)->tl_count++], (ctx)->stream); } } while (0)
#define URH_TL_RESET(ctx) do { (ctx)->tl_count = 0; } while (0)
// record events around the dense kernel when profiling is enabled
#define URH_PROF_BEGIN(ctx) do { if ((ctx)->profiling) cudaEventRecord((ctx)->ev_k0, (ctx)->stream); } while (0)
#define URH_PROF_END(ctx) do { if ((ctx)->profiling) { cudaEventRecord((ctx)->ev_k1, (ctx)->stream); (ctx)->dense_timed = 1; } } while (0)

// ---- arena ----------------------------------------------------------------------------------------
void urh_arena_reset(urh_ctx* ctx);
int urh_arena_alloc(urh_ctx* ctx, size_t bytes, void** out);
template <typename T>
static inline int urh_arena(urh_ctx* ctx, size_t count, T** out) {
    void* p = nullptr;
    int rc = urh_arena_alloc(ctx, count * sizeof(T), &p);
    *out = (T*)p;
    return rc;
}
// bump position of the arena: work that repeats per chunk releases what it took (reuse is stream-ordered, as after a reset)
struct UrhArenaMark {
    size_t block, used, live;
};
static inline UrhArenaMark urh_arena_mark(const urh_ctx* ctx) { return UrhArenaMark{ctx->arena_block, ctx->arena_used, ctx->arena_live}; }
static inline void urh_arena_release(urh_ctx* ctx, const UrhArenaMark& m) {
    ctx->arena_block = m.block;
    ctx->arena_used = m.used;
    ctx->arena_live = m.live;
}
int urh_ensure_pulses(urh_ctx* ctx, size_t rows);
// grow the pulse table to at least `rows`, keeping its first `keep` rows (a table that chunks are appended to)
int urh_ensure_pulses_keep(urh_ctx* ctx, size_t rows, size_t keep);
// streamed calls with profiling on (urh_set_profiling): lower ctx->stream_free_low to the device's free memory now (urh_stream_stats)
void urh_stream_sample_free(urh_ctx* ctx);
void urh_release_mod_plans(urh_ctx* ctx);  // modulation.cu
int urh_ensure_stage(urh_ctx* ctx, size_t bytes);

// Costas loop of a streamed PSK capture across its ring chunks (costas_spec.cu; arena memory taken before the chunks' mark):
// two {freq, phase} state slots, the summed stitch counters, the chunk layout of the first speculative chunk (0: none)
struct UrhCostasStream {
    float* state;
    int64_t* acc;
    int segs;
};
int urh_costas_stream_begin(urh_ctx* ctx, UrhCostasStream* S);
void urh_costas_shard_release(urh_ctx* ctx);
int urh_costas_stream_chunk(urh_ctx* ctx, UrhCostasStream* S, int64_t c, const void* d_iq, int dtype, int64_t n, float noise_sqrd,
                            int loop_order, float bandwidth, float* d_out);
int urh_costas_stream_end(urh_ctx* ctx, const UrhCostasStream* S);
int64_t urh_costas_arena_bytes(int64_t n, int loop_order);

// read back `count` int64 scalars from device (synchronises the ctx stream)
int urh_read_i64(urh_ctx* ctx, const int64_t* d_src, int count, int64_t* h_out);

__host__ __device__ static inline int64_t urh_div_up(int64_t a, int64_t b) { return (a + b - 1) / b; }

// (a + ib)(c + id) as std::complex<float> multiplies without -ffast-math (GCC): the naive product, and when both of its
// parts are NaN, libgcc's __mulsc3 recovery of C99 Annex G (an infinite operand gives an infinite result, not NaN).  The
// Costas loop (signal_functions.pyx:302) reaches the recovery on samples with an infinite imaginary part, fir_filter
// (signal_functions.pyx:521) on infinite samples and taps.
__device__ __forceinline__ void urh_cmulf(float a, float b, float c, float d, float& re, float& im) {
    const float ac = __fmul_rn(a, c), bd = __fmul_rn(b, d), ad = __fmul_rn(a, d), bc = __fmul_rn(b, c);
    re = __fsub_rn(ac, bd);
    im = __fadd_rn(ad, bc);
    if (isnan(re) && isnan(im)) {
        bool recalc = false;
        if (isinf(a) || isinf(b)) {
            a = copysignf(isinf(a) ? 1.0f : 0.0f, a);
            b = copysignf(isinf(b) ? 1.0f : 0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = true;
        }
        if (isinf(c) || isinf(d)) {
            c = copysignf(isinf(c) ? 1.0f : 0.0f, c);
            d = copysignf(isinf(d) ? 1.0f : 0.0f, d);
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            recalc = true;
        }
        if (!recalc && (isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc))) {
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = true;
        }
        if (recalc) {
            re = __fmul_rn(INFINITY, __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, d)));
            im = __fmul_rn(INFINITY, __fadd_rn(__fmul_rn(a, d), __fmul_rn(b, c)));
        }
    }
}

// sample size in bytes of one IQ pair for dtype
static inline int urh_iq_bytes(int dtype) {
    switch (dtype) {
        case URH_DT_I8:
        case URH_DT_U8: return 2;
        case URH_DT_I16:
        case URH_DT_U16: return 4;
        case URH_DT_F32: return 8;
        default: return 0;
    }
}

// NOISE sentinel per modulation (signal_functions.pyx:31-44)
static inline float urh_noise_value(int mod_type) {
    switch (mod_type) {
        case URH_MOD_ASK: return 0.0f;
        case URH_MOD_FSK:
        case URH_MOD_PSK:
        case URH_MOD_OQPSK: return -4.0f;
        case URH_MOD_QAM: return 0.0f * -4.0f;  // NOISE_ASK * NOISE_FSK_PSK = -0.0
        default: return 0.0f;
    }
}
