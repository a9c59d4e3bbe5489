// afp_demod (ASK/FSK), grab_pulse_lens and the fused demod+digitize path.
//
// Reference: src/urh/cythonext/signal_functions.pyx:333-378 (afp_demod), :392-495 (grab_pulse_lens).
// See dense.cuh for the dense pass and DESIGN.md for the run/candidate restatement of the digitizer.
#include "dense.cuh"
#include "scan.cuh"
#include "sparse.cuh"
#ifndef URH_FAST_MIN_BLOCKS
#define URH_FAST_MIN_BLOCKS 4
#endif
#include "fsk_fast.cuh"
#include "dense_f32.cuh"

#include <math.h>
#include <stdlib.h>

// =====================================================================================================
// Dense kernels
// =====================================================================================================

// One tile of the IQ-source dense pass: demodulate (+ optionally write qad, + optionally digitize).
template <int DT, int MOD, bool DIGITIZE>
__device__ __forceinline__ void dense_iq_tile(const void* __restrict__ iq, int64_t n, const UrhDemodParams& dp, float* __restrict__ qad_out,
                                              int vec_in, int vec_out, const UrhClassify& cls, int tol, UrhTileSummary* __restrict__ tiles,
                                              uint32_t* __restrict__ staging, int stage_cap, int16_t* __restrict__ init_cls, int cls_of_zero,
                                              int64_t tile, int has_halo, UrhTileStats* __restrict__ tile_stats, const UrhFine& fine,
                                              unsigned int* s_fine, unsigned int* g_fine) {
    const int lane = threadIdx.x & 31;
    const int64_t tile_start = tile * URH_TILE;
    const int tile_len = (int)((n - tile_start) < URH_TILE ? (n - tile_start) : URH_TILE);
    const int iters = (tile_len + 63) >> 6;

    UrhRunTracker rt;
    if (DIGITIZE) rt.init(tol, staging + tile * (int64_t)stage_cap);
    UrhStatAcc acc;
    acc.init();

    // FSK: (A, B) terms of the sample preceding the tile's first sample
    float cA = 0.0f, cB = 0.0f;
    // (a shard of a larger capture has its predecessor sample stored right before iq: has_halo)
    if (MOD == URH_MOD_FSK && (tile_start > 0 || has_halo) && lane == 0) {
        typedef typename UrhElem<DT>::type E;
        const E* pp = (const E*)iq + 2 * (tile_start - 1);
        const UrhFskTerms t = urh_fsk_terms((float)pp[0], (float)pp[1]);
        cA = t.A; cB = t.B;
    }

    UrhPair cur = urh_load_pair<DT>(iq, tile_start + 2 * lane, n, vec_in != 0);
    for (int it = 0; it < iters; it++) {
        const int64_t pos0 = tile_start + (int64_t)it * 64 + 2 * lane;
        UrhPair nxt;
        if (it + 1 < iters) nxt = urh_load_pair<DT>(iq, pos0 + 64, n, vec_in != 0);

        // noise gate: magnitude = re*re + im*im <= noise_sqrd (pyx:366-369)
        const float m0 = __fadd_rn(__fmul_rn(cur.r0, cur.r0), __fmul_rn(cur.i0, cur.i0));
        const float m1 = __fadd_rn(__fmul_rn(cur.r1, cur.r1), __fmul_rn(cur.i1, cur.i1));
        float s0 = dp.noise_value, s1 = dp.noise_value;
        if (MOD == URH_MOD_FSK) {
            const UrhFskTerms t0 = urh_fsk_terms(cur.r0, cur.i0);
            const UrhFskTerms t1 = urh_fsk_terms(cur.r1, cur.i1);
            float pA = __shfl_up_sync(URH_FULL_MASK, t1.A, 1);
            float pB = __shfl_up_sync(URH_FULL_MASK, t1.B, 1);
            if (lane == 0) { pA = cA; pB = cB; }
            cA = __shfl_sync(URH_FULL_MASK, t1.A, 31);
            cB = __shfl_sync(URH_FULL_MASK, t1.B, 31);
            if (!(m0 <= dp.noise_sqrd)) s0 = urh_fsk_angle(pA, pB, t0.C, t0.D);
            if (!(m1 <= dp.noise_sqrd)) s1 = urh_fsk_angle(t0.A, t0.B, t1.C, t1.D);
        } else if (MOD == URH_MOD_ASK) {
            if (!(m0 <= dp.noise_sqrd)) s0 = __fdiv_rn(__fsqrt_rn(m0), dp.max_mag);
            if (!(m1 <= dp.noise_sqrd)) s1 = __fdiv_rn(__fsqrt_rn(m1), dp.max_mag);
        }
        if (pos0 == 0 && !has_halo) s0 = dp.noise_value;  // result[0] = NOISE (pyx:361); shards: only the capture's first sample

        const bool v0 = pos0 < n, v1 = pos0 + 1 < n;
        if (tile_stats) {
            if (v0) { acc.add(s0); acc.all_noise = acc.all_noise && (s0 == dp.noise_value); }
            if (v1) { acc.add(s1); acc.all_noise = acc.all_noise && (s1 == dp.noise_value); }
            if (s_fine) {
                if (v0) urh_fine_add(s0, fine, s_fine, g_fine);
                if (v1) urh_fine_add(s1, fine, s_fine, g_fine);
            }
        }
        if (qad_out) {
            if (v1 && vec_out) urh_stg_f2(qad_out + pos0, s0, s1);
            else {
                if (v0) qad_out[pos0] = s0;
                if (v1) qad_out[pos0 + 1] = s1;
            }
        }
        if (DIGITIZE) {
            const int c0 = urh_classify(s0, cls), c1 = urh_classify(s1, cls);
            if (pos0 == 0) *init_cls = (int16_t)((s0 == cls.noise_value) ? -1 : cls_of_zero);
            rt.feed(it, c0, c1, v0, v1, lane);
        }
        cur = nxt;
    }
    if (tile_stats) acc.store(tile_stats + tile, lane);
    if (DIGITIZE) rt.finish(tile_len, tiles + tile, lane);
}

// IQ source, one warp per tile; fine.gh: also the fine histogram of the kept samples (dynamic shared memory URH_FINE_NB words).
template <int DT, int MOD, bool DIGITIZE>
__global__ void __launch_bounds__(URH_WARPS_PER_BLOCK * 32)
k_dense_iq(const void* __restrict__ iq, int64_t n, UrhDemodParams dp, float* __restrict__ qad_out, int vec_in,
           int vec_out, const __grid_constant__ UrhClassify cls, int tol, UrhTileSummary* __restrict__ tiles,
           uint32_t* __restrict__ staging, int stage_cap, int16_t* __restrict__ init_cls, int cls_of_zero,
           int64_t tile_begin, int64_t tile_count, int has_halo, UrhTileStats* __restrict__ tile_stats, const UrhFine fine) {
    extern __shared__ unsigned int s_fine[];   // [URH_FINE_NB] when fine.gh
    const int64_t tile_rel = (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK + (threadIdx.x >> 5);
    const int64_t block_tile0 = tile_begin + (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK;
    if (fine.gh) urh_fine_zero(s_fine);
    if (tile_rel < tile_count && (tile_begin + tile_rel) * URH_TILE < n)
        dense_iq_tile<DT, MOD, DIGITIZE>(iq, n, dp, qad_out, vec_in, vec_out, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero,
                                    tile_begin + tile_rel, has_halo, tile_stats, fine,
                                    fine.gh ? s_fine : nullptr, fine.gh ? urh_fine_row(fine, tile_begin + tile_rel, block_tile0) : nullptr);
    if (fine.gh) urh_fine_flush(fine, s_fine, block_tile0);
}

// Fast kernel: full, aligned, order-2 FSK tiles [tile_begin, tile_begin + tile_count), tile_begin >= 1
// (fsk_fast.cuh: float2-paired math, same bits as the generic kernel).
template <int DT, bool DIGITIZE, bool WRITE, bool STATS>
__global__ void __launch_bounds__(URH_WARPS_PER_BLOCK * 32, URH_FAST_MIN_BLOCKS)
k_fsk_fast(const void* __restrict__ iq, int64_t n, UrhDemodParams dp, float* __restrict__ qad_out, float thr0,
           float cls_noise, int tol, UrhTileSummary* __restrict__ tiles, uint32_t* __restrict__ staging, int stage_cap,
           int64_t tile_begin, int64_t tile_count, UrhTileStats* __restrict__ tile_stats, const UrhFine fine) {
    extern __shared__ unsigned int s_fine[];   // [URH_FINE_NB] when STATS and fine.gh
    const bool fine_on = STATS && fine.gh;
    const int lane = threadIdx.x & 31;
    const int64_t tile_rel = (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK + (threadIdx.x >> 5);
    const int64_t block_tile0 = tile_begin + (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK;
    if (fine_on) urh_fine_zero(s_fine);
    if (tile_rel < tile_count) {
        const int64_t tile = tile_begin + tile_rel;
        UrhRunTracker rt;
        if (DIGITIZE) rt.init(tol, staging + tile * (int64_t)stage_cap);
        UrhOne one;
        one.p = dp.one;
        one.m = dp.mone;
        urh_fsk_full_tile<DT, DIGITIZE, WRITE, STATS>(iq, n, tile * URH_TILE, dp, qad_out, thr0, cls_noise, rt, lane, one,
                                                      STATS ? tile_stats + tile : nullptr, 0u, DIGITIZE ? tiles + tile : nullptr, fine,
                                                      fine_on ? s_fine : nullptr, fine_on ? urh_fine_row(fine, tile, block_tile0) : nullptr);
    }
    if (fine_on) urh_fine_flush(fine, s_fine, block_tile0);
}

// The same kernel with the input staged through the shared-memory FIFO.
// DIGITIZE and STATS: the speculative pass of the detect-center step; the threshold is the guess *d_thr0, margin[tile] its proof.
#define URH_FSK_FIFO 3
template <int DT, bool DIGITIZE, bool WRITE, bool STATS>
__global__ void __launch_bounds__(URH_WARPS_PER_BLOCK * 32, (DT == URH_DT_F32) ? 5 : 4)   // (the integer variants spill at 48 registers)
k_fsk_fifo(const void* __restrict__ iq, int64_t n, UrhDemodParams dp, float* __restrict__ qad_out, float thr0,
           float cls_noise, int tol, UrhTileSummary* __restrict__ tiles, uint32_t* __restrict__ staging, int stage_cap,
           int64_t tile_begin, int64_t tile_count, UrhTileStats* __restrict__ tile_stats, const UrhFine fine,
           const float* __restrict__ d_thr0 = nullptr, float* __restrict__ margin = nullptr) {
    __shared__ __align__(16) unsigned char s_fifo[URH_WARPS_PER_BLOCK][URH_FSK_FIFO + 1][64 * 2 * sizeof(typename UrhElem<DT>::type)];
    extern __shared__ unsigned int s_fine[];   // [URH_FINE_NB] when STATS and fine.gh
    const bool fine_on = STATS && fine.gh;
    if (DIGITIZE && STATS) thr0 = *d_thr0;
    const int lane = threadIdx.x & 31;
    const int64_t tile_rel = (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK + (threadIdx.x >> 5);
    const int64_t block_tile0 = tile_begin + (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK;
    if (fine_on) urh_fine_zero(s_fine);
    if (tile_rel < tile_count) {
        const int64_t tile = tile_begin + tile_rel;
        UrhRunTracker rt;
        if (DIGITIZE) rt.init(tol, staging + tile * (int64_t)stage_cap);
        UrhOne one;
        one.p = dp.one;
        one.m = dp.mone;
        const uint32_t fifo = (uint32_t)__cvta_generic_to_shared(&s_fifo[threadIdx.x >> 5][0][0]);
        urh_fsk_full_tile<DT, DIGITIZE, WRITE, STATS, URH_FSK_FIFO>(iq, n, tile * URH_TILE, dp, qad_out, thr0, cls_noise, rt, lane, one,
                                                                    STATS ? tile_stats + tile : nullptr, fifo,
                                                                    DIGITIZE ? tiles + tile : nullptr, fine, fine_on ? s_fine : nullptr,
                                                                    fine_on ? urh_fine_row(fine, tile, block_tile0) : nullptr,
                                                                    (DIGITIZE && STATS) ? margin + tile : nullptr);
    }
    if (fine_on) urh_fine_flush(fine, s_fine, block_tile0);
}

// Threshold guess t_g of the speculative detect-center step (float32 FSK captures, DESIGN.md §4.4.1).  One block demodulates
// URH_GUESS_SAMPLES samples spread evenly over the capture (the same noise gate, plain atan2f), histograms the kept ones over
// URH_GUESS_BINS bins spanning their [min, max], and takes the midpoint of the two most populated local maxima - the rule
// k_center_pick applies to the capture's histogram.  The mean of the kept samples would not do: with one symbol dominating it sits
// next to that symbol's level.  One peak: its bin; none: the middle of the range.  Only the step's speed depends on the guess.
// forced != 0 replaces the guess by forced_tg ($URH_B200_SPECULATE_GUESS).  Also zeroes the redo counter.
#define URH_GUESS_SAMPLES 16384
#define URH_GUESS_BINS 128
#define URH_GUESS_THREADS 1024
__global__ void __launch_bounds__(URH_GUESS_THREADS) k_speculate_guess(const float2* __restrict__ iq, int64_t n, float noise_sqrd, int forced,
                                                                      float forced_tg, float* __restrict__ d_tg, unsigned int* __restrict__ redone) {
    constexpr int PER = URH_GUESS_SAMPLES / URH_GUESS_THREADS;
    __shared__ unsigned int s_hist[URH_GUESS_BINS];
    __shared__ float s_mn[32], s_mx[32];
    if (forced) {
        if (threadIdx.x == 0) { *d_tg = forced_tg; *redone = 0u; }
        return;
    }
    for (int b = threadIdx.x; b < URH_GUESS_BINS; b += blockDim.x) s_hist[b] = 0u;
    float v[PER];
    float mn = INFINITY, mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < PER; k++) {
        const int64_t i = 1 + (int64_t)(k * URH_GUESS_THREADS + threadIdx.x) * (n - 1) / URH_GUESS_SAMPLES;   // 1 .. n - 1
        const float2 p = iq[i - 1], c = iq[i];
        v[k] = NAN;   // gated
        if (!(c.x * c.x + c.y * c.y <= noise_sqrd)) {
            v[k] = atan2f(p.x * c.y - p.y * c.x, p.x * c.x + p.y * c.y);
            mn = fminf(mn, v[k]);
            mx = fmaxf(mx, v[k]);
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(URH_FULL_MASK, mn, off));
        mx = fmaxf(mx, __shfl_xor_sync(URH_FULL_MASK, mx, off));
    }
    if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    mn = INFINITY; mx = -INFINITY;
    for (int w = 0; w < URH_GUESS_THREADS / 32; w++) { mn = fminf(mn, s_mn[w]); mx = fmaxf(mx, s_mx[w]); }
    const float width = (mx - mn) / URH_GUESS_BINS;   // mn > mx (nothing kept) or width 0: no histogram
    if (width > 0.0f) {
#pragma unroll
        for (int k = 0; k < PER; k++)
            if (!isnan(v[k])) atomicAdd(&s_hist[min((int)((v[k] - mn) / width), URH_GUESS_BINS - 1)], 1u);
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    *redone = 0u;
    if (!(mn <= mx)) { *d_tg = 0.0f; return; }
    if (!(width > 0.0f)) { *d_tg = mn; return; }
    constexpr int WINDOW = (int)(0.05 * URH_GUESS_BINS) + 1;
    int top[2] = {-1, -1};
    for (int b = 0; b < URH_GUESS_BINS; b++) {
        const unsigned int y = s_hist[b];
        bool peak = y > 0u;
        for (int d = 1; d < WINDOW && peak; d++)
            peak = y > (b + d < URH_GUESS_BINS ? s_hist[b + d] : 0u) && y > (b - d >= 0 ? s_hist[b - d] : 0u);
        if (!peak) continue;
        if (top[0] < 0 || y > s_hist[top[0]]) { top[1] = top[0]; top[0] = b; }
        else if (top[1] < 0 || y > s_hist[top[1]]) top[1] = b;
    }
    if (top[0] < 0) *d_tg = 0.5f * (mn + mx);
    else if (top[1] < 0) *d_tg = mn + ((float)top[0] + 0.5f) * width;
    else *d_tg = mn + (0.5f * (float)(top[0] + top[1]) + 0.5f) * width;
}

// =====================================================================================================
// Host side
// =====================================================================================================

extern "C" int urh_get_center_thresholds(float center, float spacing, int modulation_order, float* h_out) {
    // signal_functions.pyx:380-390 — float32 arithmetic on (int * float)
    const int n = modulation_order / 2;
    for (int i = 0; i < n; i++) {
        volatile float t = (float)(n - (i + 1)) * spacing;
        h_out[i] = center - t;
    }
    for (int i = n; i < modulation_order - 1; i++) {
        volatile float t = (float)(i + 1 - n) * spacing;
        h_out[i] = center + t;
    }
    return URH_OK;
}

static int fill_classify(urh_ctx* ctx, UrhClassify* C, int mod_type, float center, uint8_t bits_per_symbol,
                         float spacing) {
    if (bits_per_symbol > 8) URH_FAIL(ctx, URH_ERR_INVALID, "bits_per_symbol %d > 8 not supported", (int)bits_per_symbol);
    memset(C, 0, sizeof(*C));
    C->noise_value = urh_noise_value(mod_type);
    C->order = 1 << bits_per_symbol;
    if (C->order > 1) urh_get_center_thresholds(center, spacing, C->order, C->thr);
    return URH_OK;
}

static int host_classify(float s, const UrhClassify& C) {
    int c = C.order - 1;
    for (int k = 0; k < C.order - 1; k++)
        if (s <= C.thr[k]) { c = k; break; }
    return c;
}

static float max_magnitude_for(int dtype) {
    // signal_functions.pyx:343-352: double sqrt of an integer constant, stored in a float
    switch (dtype) {
        case URH_DT_I8: return (float)sqrt(127.0 * 127.0 + 128.0 * 128.0);
        case URH_DT_U8: return (float)sqrt(255.0 * 255.0);
        case URH_DT_I16: return (float)sqrt(32768.0 * 32768.0 + 32767.0 * 32767.0);
        case URH_DT_U16: return (float)sqrt(65535.0 * 65535.0);
        default: return (float)sqrt(2.0);
    }
}

static bool iq_vec_aligned(const void* p, int dtype) { return ((uintptr_t)p % (2 * (size_t)urh_iq_bytes(dtype))) == 0; }

// tile_lo / tile_hi: restrict the pass to tiles [tile_lo, tile_hi) (chunked ingest: a chunk is demodulated as soon as its
// upload has landed); tile_hi < 0 = all tiles.
// spec != NULL (float32 FSK, tile statistics, no DIG): the fast kernel's tiles are also digitized at the guess spec->tg into
// tiles / staging (tol, stage_cap), with their margins; spec->lo / hi is set to that tile range (UrhSpec).
template <int DT, int MOD, bool DIG>
static int launch_dense_iq_t(urh_ctx* ctx, const void* d_iq, int64_t n, const UrhDemodParams& dp, float* d_qad,
                             const UrhClassify& cls, int tol, UrhTileSummary* tiles, uint32_t* staging,
                             int stage_cap, int16_t* init_cls, int cls_of_zero, int has_halo = 0,
                             UrhTileStats* tile_stats = nullptr, int64_t tile_lo = 0, int64_t tile_hi = -1,
                             const UrhFine& fine = UrhFine{}, UrhSpec* spec = nullptr) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const size_t fine_smem = fine.gh ? (size_t)URH_FINE_NB * sizeof(unsigned int) : 0;
    if (tile_hi < 0 || tile_hi > ntiles) tile_hi = ntiles;
    const int vec_in = iq_vec_aligned(d_iq, DT) ? 1 : 0;
    const int vec_out = (d_qad && ((uintptr_t)d_qad % 8) == 0) ? 1 : 0;
    const int threads = URH_WARPS_PER_BLOCK * 32;
    auto generic = [&](int64_t begin, int64_t end) -> int {   // tiles [begin, end) clipped to the requested range
        begin = begin < tile_lo ? tile_lo : begin;
        end = end > tile_hi ? tile_hi : end;
        const int64_t count = end - begin;
        if (count <= 0) return URH_OK;
        URH_LAUNCH(ctx, (k_dense_iq<DT, MOD, DIG>), (unsigned)urh_div_up(count, URH_WARPS_PER_BLOCK), threads, fine_smem, d_iq, n, dp,
                   d_qad, vec_in, vec_out, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, begin, count, has_halo,
                   tile_stats, fine);
        return URH_OK;
    };
    // FSK on aligned buffers with a binary digitizer: tiles 1 .. nfull-1 take the paired fast kernel
    const int64_t nfull = n / URH_TILE;
    const bool fast = MOD == URH_MOD_FSK && vec_in && (!d_qad || vec_out) && (!DIG || cls.order == 2) && nfull > 1;
    URH_PROF_BEGIN(ctx);
    if (fast) {
        const int64_t fb = tile_lo > 1 ? tile_lo : 1, fe = tile_hi < nfull ? tile_hi : nfull;
        if (fe > fb) {
            const unsigned grid = (unsigned)urh_div_up(fe - fb, URH_WARPS_PER_BLOCK);
            // the variant that stages its input through the shared-memory FIFO (URH_B200_FSK_NO_FIFO selects the register-fed loop)
            static const bool fifo = getenv("URH_B200_FSK_NO_FIFO") == nullptr;
            const bool ff = fifo;
            bool speculated = false;
            if constexpr (DT == URH_DT_F32 && MOD == URH_MOD_FSK && !DIG) {
                if (spec && ff && tile_stats && d_qad) {
                    URH_LAUNCH(ctx, (k_fsk_fifo<DT, true, true, true>), grid, threads, fine_smem, d_iq, n, dp, d_qad, 0.0f, dp.noise_value,
                               tol, tiles, staging, stage_cap, fb, fe - fb, tile_stats, fine, (const float*)spec->tg, spec->margin);
                    spec->lo = fb;
                    spec->hi = fe;
                    speculated = true;
                }
            }
            if (speculated) {
            } else if (tile_stats && d_qad && !DIG) {
                if (ff) URH_LAUNCH(ctx, (k_fsk_fifo<DT, false, true, true>), grid, threads, fine_smem, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value,
                                   tol, tiles, staging, stage_cap, fb, fe - fb, tile_stats, fine);
                else URH_LAUNCH(ctx, (k_fsk_fast<DT, false, true, true>), grid, threads, fine_smem, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value,
                                tol, tiles, staging, stage_cap, fb, fe - fb, tile_stats, fine);
            } else if (d_qad) {
                if (ff) URH_LAUNCH(ctx, (k_fsk_fifo<DT, DIG, true, false>), grid, threads, 0, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value, tol,
                                   tiles, staging, stage_cap, fb, fe - fb, nullptr, UrhFine{});
                else URH_LAUNCH(ctx, (k_fsk_fast<DT, DIG, true, false>), grid, threads, 0, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value, tol,
                                tiles, staging, stage_cap, fb, fe - fb, nullptr, UrhFine{});
            } else {
                if (ff) URH_LAUNCH(ctx, (k_fsk_fifo<DT, DIG, false, false>), grid, threads, 0, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value, tol,
                                   tiles, staging, stage_cap, fb, fe - fb, nullptr, UrhFine{});
                else URH_LAUNCH(ctx, (k_fsk_fast<DT, DIG, false, false>), grid, threads, 0, d_iq, n, dp, d_qad, cls.thr[0], cls.noise_value, tol,
                                tiles, staging, stage_cap, fb, fe - fb, nullptr, UrhFine{});
            }
        }
        URH_CHECK(generic(0, 1));
        URH_CHECK(generic(nfull, ntiles));
    } else {
        URH_CHECK(generic(0, ntiles));
    }
    URH_PROF_END(ctx);
    return URH_OK;
}

template <int MOD, bool DIG>
static int launch_dense_iq_m(urh_ctx* ctx, int dtype, const void* d_iq, int64_t n, const UrhDemodParams& dp,
                             float* d_qad, const UrhClassify& cls, int tol, UrhTileSummary* tiles,
                             uint32_t* staging, int stage_cap, int16_t* init_cls, int cls_of_zero, int has_halo = 0,
                             UrhTileStats* tile_stats = nullptr, int64_t tile_lo = 0, int64_t tile_hi = -1,
                             const UrhFine& fine = UrhFine{}, UrhSpec* spec = nullptr) {
    switch (dtype) {
        case URH_DT_I8: return launch_dense_iq_t<URH_DT_I8, MOD, DIG>(ctx, d_iq, n, dp, d_qad, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, has_halo, tile_stats, tile_lo, tile_hi, fine);
        case URH_DT_U8: return launch_dense_iq_t<URH_DT_U8, MOD, DIG>(ctx, d_iq, n, dp, d_qad, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, has_halo, tile_stats, tile_lo, tile_hi, fine);
        case URH_DT_I16: return launch_dense_iq_t<URH_DT_I16, MOD, DIG>(ctx, d_iq, n, dp, d_qad, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, has_halo, tile_stats, tile_lo, tile_hi, fine);
        case URH_DT_U16: return launch_dense_iq_t<URH_DT_U16, MOD, DIG>(ctx, d_iq, n, dp, d_qad, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, has_halo, tile_stats, tile_lo, tile_hi, fine);
        case URH_DT_F32: return launch_dense_iq_t<URH_DT_F32, MOD, DIG>(ctx, d_iq, n, dp, d_qad, cls, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, has_halo, tile_stats, tile_lo, tile_hi, fine, spec);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    }
}

int urh_costas_demod(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_sqrd, int loop_order,
                     float bandwidth, float* d_out);  // costas.cu

static UrhDemodParams make_demod_params(float noise_mag, int mod_type, int dtype) {
    UrhDemodParams dp;
    volatile float nm = noise_mag;
    volatile float sq = nm * nm;
    dp.noise_sqrd = sq;
    dp.noise_value = urh_noise_value(mod_type);
    dp.max_mag = max_magnitude_for(dtype);
    dp.one = 1.0f;
    dp.mone = -1.0f;
    return dp;
}

extern "C" int urh_afp_demod(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                             int mod_order, float costas_loop_bandwidth, float* d_out) {
    if (n < 0) URH_FAIL(ctx, URH_ERR_INVALID, "negative length");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (n == 0) return URH_OK;
    if (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK && mod_type != URH_MOD_PSK)) {
        // pyx:335-336 (short input) and pyx:360,371-376 (unknown mod_type leaves zeros, result[0] = NOISE)
        URH_CUDA(ctx, cudaMemsetAsync(d_out, 0, (size_t)n * sizeof(float), ctx->stream));
        if (n > 2) {
            const float nv = urh_noise_value(mod_type);
            URH_CUDA(ctx, cudaMemcpyAsync(d_out, &nv, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
            URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
        return URH_OK;
    }
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    if (mod_type == URH_MOD_PSK) return urh_costas_demod(ctx, d_iq, dtype, n, dp.noise_sqrd, mod_order, costas_loop_bandwidth, d_out);
    UrhClassify cls;
    memset(&cls, 0, sizeof(cls));
    if (mod_type == URH_MOD_ASK)
        return launch_dense_iq_m<URH_MOD_ASK, false>(ctx, dtype, d_iq, n, dp, d_out, cls, 0, nullptr, nullptr, 0, nullptr, 0);
    return launch_dense_iq_m<URH_MOD_FSK, false>(ctx, dtype, d_iq, n, dp, d_out, cls, 0, nullptr, nullptr, 0, nullptr, 0);
}

int urh_center_tiles_begin(urh_ctx* ctx, const float* d_x, const UrhTileStats* ts, int64_t n, int64_t* h_total);  // center.cu

// afp_demod (ASK / FSK) that also collects, in the same pass over the IQ samples, what detect_center needs: per-tile
// {count, min, max, sum, sumsq} of the samples it keeps (> -4).  *h_kept = number of kept samples.  The table stays in
// the ctx arena for urh_center_window_stats / urh_center_histogram_tiles (any other ctx call invalidates it).
// halo = 1: the sample preceding d_iq (the previous shard's last) is readable right before it, so qad[0] is a real value
// instead of the capture-start NOISE sentinel.
extern "C" int urh_afp_demod_tiles(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                   float* d_qad_out, int halo, int64_t* h_kept) {
    if (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) || !d_qad_out)
        URH_FAIL(ctx, URH_ERR_INVALID, "urh_afp_demod_tiles: ASK/FSK, n > 2 and a qad buffer are required");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    urh_arena_reset(ctx);
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    UrhClassify cls;
    memset(&cls, 0, sizeof(cls));
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    UrhTileStats* ts;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &ts));
    if (mod_type == URH_MOD_ASK)
        URH_CHECK((launch_dense_iq_m<URH_MOD_ASK, false>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, 0, nullptr, nullptr, 0, nullptr, 0, halo, ts)));
    else
        URH_CHECK((launch_dense_iq_m<URH_MOD_FSK, false>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, 0, nullptr, nullptr, 0, nullptr, 0, halo, ts)));
    return urh_center_tiles_begin(ctx, d_qad_out, ts, n, h_kept);
}

// Shared tail of the two digitizer entry points: tile table + staging -> merged (state, length) rows.
int urh_finish_local(urh_ctx* ctx, int64_t n, int tol, bool is_ask, uint32_t sps, const UrhTileSummary* tiles, const uint32_t* staging,
                     int stage_cap, const int16_t* d_init, int64_t* k);   // finish.cu
int urh_finish_shard(urh_ctx* ctx, int64_t n, int tol, bool is_ask, uint32_t sps, const UrhTileSummary* tiles, const uint32_t* staging,
                     int stage_cap, const int16_t* d_init, int64_t global_offset, int64_t n_total, int64_t* k);   // finish.cu

static int digitize_finish(urh_ctx* ctx, int64_t n, int tol, bool is_ask, uint32_t sps, UrhTileSummary* tiles,
                           uint32_t* staging, int stage_cap, int16_t* d_init, int64_t* k) {
    if (getenv("URH_B200_OLD_FINISH")) {   // the candidate-table formulation (kept for the segmenter; A/B switch for measurements)
        UrhCandidates cand;
        URH_CHECK(urh_collect_candidates(ctx, n, tol, tiles, staging, stage_cap, &cand));
        return urh_pulses_from_candidates(ctx, n, tol, is_ask, sps, cand, d_init, k);
    }
    return urh_finish_local(ctx, n, tol, is_ask, sps, tiles, staging, stage_cap, d_init, k);
}

static int stage_cap_for(int tol) { return URH_TILE / (tol + 1) + 2; }

extern "C" int urh_grab_pulse_lens(urh_ctx* ctx, const float* d_qad, int64_t n, float center, uint16_t tolerance,
                                   int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                                   float center_spacing, int64_t* k) {
    if (!k) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    if (n < 0) URH_FAIL(ctx, URH_ERR_INVALID, "negative length");
    if (n == 0) return URH_OK;  // pyx:416-417 -> empty (0,2) table
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const int tol = tolerance;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    const unsigned grid = (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK);
    const int vec_in = (((uintptr_t)d_qad % 8) == 0) ? 1 : 0;
    URH_PROF_BEGIN(ctx);
    if (cls.order == 2)
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad, n, vec_in, cls, tol, tiles,
                   staging, cap, d_init, host_classify(0.0f, cls));
    else
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad, n, vec_in, cls, tol, tiles,
                   staging, cap, d_init, host_classify(0.0f, cls));
    URH_PROF_END(ctx);
    return digitize_finish(ctx, n, tol, mod_type == URH_MOD_ASK, samples_per_symbol, tiles, staging, cap, d_init, k);
}

extern "C" int urh_demod_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag,
                                  int mod_type, float center, uint16_t tolerance, uint32_t samples_per_symbol,
                                  uint8_t bits_per_symbol, float center_spacing, float* d_qad_out, int64_t* k) {
    if (!k) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    if (n < 0) URH_FAIL(ctx, URH_ERR_INVALID, "negative length");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (n == 0) return URH_OK;
    if (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK)) {
        // not a fusable case: run the two reference steps back to back (PSK is a serial recurrence)
        float* q = d_qad_out;
        if (!q) URH_CUDA(ctx, cudaMalloc((void**)&q, (size_t)n * sizeof(float)));
        int rc = urh_afp_demod(ctx, d_iq, dtype, n, noise_mag, mod_type, 1 << bits_per_symbol, 0.1f, q);
        if (rc == URH_OK)
            rc = urh_grab_pulse_lens(ctx, q, n, center, tolerance, mod_type, samples_per_symbol, bits_per_symbol,
                                     center_spacing, k);
        if (!d_qad_out) {
            cudaStreamSynchronize(ctx->stream);
            cudaFree(q);
        }
        return rc;
    }
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    const int tol = tolerance;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    const int c0 = host_classify(0.0f, cls);
    if (mod_type == URH_MOD_ASK)
        URH_CHECK((launch_dense_iq_m<URH_MOD_ASK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0)));
    else
        URH_CHECK((launch_dense_iq_m<URH_MOD_FSK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0)));
    return digitize_finish(ctx, n, tol, mod_type == URH_MOD_ASK, samples_per_symbol, tiles, staging, cap, d_init, k);
}

// =====================================================================================================
// Sharded captures (SURVEY §8e): one contiguous sample range per GPU, 1-sample halo for the FSK conjugate
// product, run-carry descriptors exchanged between ranks, candidate tables gathered to one rank.
// =====================================================================================================
// Step 1 on every rank.  d_iq points at the shard's first own sample; when has_halo != 0 the sample that precedes
// the shard in the capture is stored immediately before it (d_iq[-1]).  Keeps the tile table in the arena for step 2.
// h_summary = {last_cls, last_len, whole, init_cls}: the shard's closing run and (rank 0) the digitizer's initial state.
extern "C" int urh_shard_dense(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag, int mod_type,
                               float center, uint16_t tolerance, uint8_t bits_per_symbol, float center_spacing,
                               float* d_qad_out, int64_t* h_summary) {
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "empty shard");
    if (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) URH_FAIL(ctx, URH_ERR_INVALID, "sharded path: ASK / FSK only (PSK is a serial recurrence)");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    const int tol = tolerance;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
    const int c0 = host_classify(0.0f, cls);
    if (mod_type == URH_MOD_ASK)
        URH_CHECK((launch_dense_iq_m<URH_MOD_ASK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0, has_halo)));
    else
        URH_CHECK((launch_dense_iq_m<URH_MOD_FSK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0, has_halo)));
    ctx->shard_tiles = tiles;
    ctx->shard_staging = staging;
    ctx->shard_cap = cap;
    ctx->shard_n = n;
    ctx->shard_tol = tol;
    URH_CHECK(urh_shard_run_total(ctx, n, tiles, h_summary));
    int16_t init16 = 0;
    URH_CUDA(ctx, cudaMemcpyAsync(&init16, d_init, sizeof(int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h_summary[3] = init16;
    return URH_OK;
}

// Step 1 for a shard that is already demodulated (the center became known only after the demodulation pass): the
// digitizer's dense pass over qad.  Classification is per sample, so no halo is involved; same h_summary as urh_shard_dense.
extern "C" int urh_shard_dense_qad(urh_ctx* ctx, const float* d_qad, int64_t n, int mod_type, float center, uint16_t tolerance,
                                   uint8_t bits_per_symbol, float center_spacing, int64_t* h_summary) {
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "empty shard");
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const int tol = tolerance;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
    const int vec_in = (((uintptr_t)d_qad % 8) == 0) ? 1 : 0;
    URH_PROF_BEGIN(ctx);
    const unsigned grid = (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK);
    if (cls.order == 2)
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad, n, vec_in, cls, tol, tiles, staging, cap,
                   d_init, host_classify(0.0f, cls));
    else
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad, n, vec_in, cls, tol, tiles, staging, cap,
                   d_init, host_classify(0.0f, cls));
    URH_PROF_END(ctx);
    ctx->shard_tiles = tiles;
    ctx->shard_staging = staging;
    ctx->shard_cap = cap;
    ctx->shard_n = n;
    ctx->shard_tol = tol;
    URH_CHECK(urh_shard_run_total(ctx, n, tiles, h_summary));
    int16_t init16 = 0;
    URH_CUDA(ctx, cudaMemcpyAsync(&init16, d_init, sizeof(int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h_summary[3] = init16;
    return URH_OK;
}

// ---- streaming through a ring of device slots (DESIGN.md §4.11) -----------------------------------------------------------------
// A chunk is a whole number of tiles (the last one excepted), so every tile has the bounds and the arithmetic it has in the resident
// call.  IQ kernels see the slot through a pointer shifted back by the chunk's first sample: they index the capture globally, their
// tile range is the chunk's, and the halo sample (uploaded with the chunk) sits where the resident buffer holds it.
int urh_finish_chunk(urh_ctx* ctx, int64_t n, int tol, bool is_ask, uint32_t sps, const UrhTileSummary* tiles, const uint32_t* staging,
                     int stage_cap, const int16_t* d_init, UrhChain* chain, int64_t global_offset, int64_t n_total, int64_t row_base,
                     int64_t rows_cap, int64_t* k);   // finish.cu

#define URH_STREAM_MAX_RING 8
#define URH_STREAM_PAD 256   // slot = [pad][halo][chunk]: the chunk starts 256 bytes in, the halo sample right before it
enum { URH_OP_UPLOAD = 0, URH_OP_COMPUTE = 1, URH_OP_DOWNLOAD = 2 };

static int64_t stream_chunk_samples(int64_t n, int64_t cs) {
    if (cs <= 0) cs = (int64_t)1 << 24;
    cs -= cs % URH_TILE;
    if (cs < URH_TILE) cs = URH_TILE;
    const int64_t whole = urh_div_up(n > 0 ? n : 1, URH_TILE) * URH_TILE;   // a capture shorter than a chunk: one slot of its size
    return cs < whole ? cs : whole;
}
// rows one digitizer pass over n samples can produce: firings are >= tol + 1 samples apart, plus the head and the tail row
static int64_t rows_bound(int64_t n, int tol) { return n / (tol + 1) + 3; }

// Op semantics (the driver below and tests/test_stream_plan_cpu.py's model):
//   upload(c, s)   copy stream 0: waits for the last compute recorded on slot s, copies, records "uploaded" on s
//   compute(c, s)  compute stream: waits for "uploaded" on s (uploading calls) and for the last download recorded on s (downloading
//                  calls), runs the chunk, records "computed" on s
//   download(c, s) copy stream 1: waits for "computed" on s, copies qad out, records "downloaded" on s
// Uploads run R - 1 chunks ahead: the upload of chunk c + R - 1 is issued before compute(c), into the slot compute(c - 1) released.
extern "C" int urh_stream_schedule(int64_t n, int64_t chunk_samples, int ring, int flags, int64_t* h_ops, int64_t cap, int64_t* count) {
    if (!count || n < 0 || ring < 2 || ring > URH_STREAM_MAX_RING) return URH_ERR_INVALID;
    const int64_t cs = stream_chunk_samples(n, chunk_samples);
    const int64_t chunks = urh_div_up(n, cs);
    const bool up = flags & URH_STREAM_UPLOAD, down = flags & URH_STREAM_DOWNLOAD, halo = flags & URH_STREAM_HALO;
    int64_t k = 0;
    auto emit = [&](int64_t kind, int64_t c) {
        if (h_ops && k < cap) {
            int64_t* o = h_ops + 6 * k;
            o[0] = kind; o[1] = c; o[2] = c % ring; o[3] = c * cs; o[4] = (c + 1) * cs < n ? (c + 1) * cs : n;
            o[5] = (kind == URH_OP_UPLOAD && halo && c > 0) ? 1 : 0;
        }
        k++;
    };
    if (up)
        for (int64_t c = 0; c < ring - 1 && c < chunks; c++) emit(URH_OP_UPLOAD, c);
    for (int64_t c = 0; c < chunks; c++) {
        if (up && c + ring - 1 < chunks) emit(URH_OP_UPLOAD, c + ring - 1);
        emit(URH_OP_COMPUTE, c);
        if (down) emit(URH_OP_DOWNLOAD, c);
    }
    *count = k;
    return (h_ops && k > cap) ? URH_ERR_INVALID : URH_OK;
}

// Device bytes of the ring (one cudaMallocAsync block) and of the arena requests of a call; the one place these sizes live.
struct StreamSizes {
    int64_t cs;          // chunk samples
    int64_t src_slot;    // bytes per source slot (0: no upload ring)
    int64_t qad_slot;    // bytes per qad slot (0: no download ring)
    int64_t ring_bytes;  // the ring block
    int64_t arena;       // arena requests (tiles, staging, carries, finish, center tables)
    int64_t scan_items;  // largest table a look-back scan of the call runs over
    int64_t rows_chunk;  // bound of one chunk's rows
};
static int64_t r256(int64_t b) { return (b + 255) & ~(int64_t)255; }
static int64_t finish_arena_bytes(int64_t tiles, int64_t rows_cap, bool ask) {
    return r256(tiles * (int64_t)sizeof(RunCarry)) + 2 * r256(tiles * 4) + 2 * r256(tiles * 8) + r256((32 + 8) * 8) +
           (ask ? r256(rows_cap * 16) : 0);
}
// loop order of a PSK footprint entry (0: not PSK)
static int psk_order_of(int entry) { return (entry & URH_STREAM_PSK) ? ((entry & URH_STREAM_PSK4) ? 4 : 2) : 0; }
static int psk_entry_flags(int mod_order) { return URH_STREAM_PSK | (mod_order >= 4 ? URH_STREAM_PSK4 : 0); }

static StreamSizes stream_sizes(int64_t n, int dtype, int tol, int64_t chunk_samples, int ring, int entry) {
    StreamSizes z;
    const int kind = entry & 0xf;
    const int psk = psk_order_of(entry);
    const bool resident = entry & URH_STREAM_RESIDENT;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    z.cs = resident ? ntiles * URH_TILE : stream_chunk_samples(n, chunk_samples);
    const int64_t ct = z.cs / URH_TILE;
    const int64_t cap = stage_cap_for(tol);
    const bool iq = kind != URH_STREAM_ENTRY_GRAB_PULSE_LENS;
    const bool digitize = kind != URH_STREAM_ENTRY_AFP_DEMOD;
    z.rows_chunk = rows_bound(z.cs, tol);
    if (resident) {   // what the resident entry allocates for a host capture: the capture and qad on the device, full-size tables
        z.src_slot = iq ? n * urh_iq_bytes(dtype) : n * 4;
        z.qad_slot = (kind == URH_STREAM_ENTRY_GRAB_PULSE_LENS) ? 0 : n * 4;
        z.ring_bytes = r256(z.src_slot) + r256(z.qad_slot);
    } else {
        z.src_slot = (kind == URH_STREAM_ENTRY_GRAB_PULSE_LENS && (entry & URH_STREAM_QAD_ON_DEVICE)) ? 0
                     : URH_STREAM_PAD + z.cs * (iq ? urh_iq_bytes(dtype) : 4);
        // PSK digitizing reads each chunk's qad from a device slot, downloaded or not
        const bool qad_ring = kind == URH_STREAM_ENTRY_AFP_DEMOD ||
                              (kind == URH_STREAM_ENTRY_DEMOD_DIGITIZE && ((entry & URH_STREAM_QAD_OUT) || psk));
        z.qad_slot = qad_ring ? z.cs * 4 : 0;
        z.ring_bytes = ring * (r256(z.src_slot) + r256(z.qad_slot));
        if (kind == URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE) z.ring_bytes += r256(n * 4);   // resident qad (the caller's buffer)
    }
    z.arena = 0;
    z.scan_items = ct > z.rows_chunk ? ct : z.rows_chunk;
    if (digitize) z.arena += r256(ct * (int64_t)sizeof(UrhTileSummary)) + r256(ct * cap * 4) + r256(16) + r256(sizeof(UrhChain)) +
                             finish_arena_bytes(ct, z.rows_chunk, true);
    // the Costas loop's tables for one chunk, the state slots and the summed counters (costas_spec.cu)
    if (psk && !resident) z.arena += urh_costas_arena_bytes(z.cs, psk) + r256(16) + r256(6 * 8);
    if (kind == URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE) {   // tile statistics, fine histogram, center chain (center.cu)
        z.arena += r256(ntiles * (int64_t)sizeof(UrhTileStats)) + r256((int64_t)URH_FINE_SLABS * URH_FINE_NB * 4) + r256((ntiles + 1) * 8) +
                   ((int64_t)2 << 20);
        if (ntiles > z.scan_items) z.scan_items = ntiles;
    }
    return z;
}

extern "C" int urh_stream_footprint(int64_t n, int dtype, int tolerance, int64_t chunk_samples, int ring, int entry, int64_t rows,
                                    int64_t* bytes) {
    if (!bytes || n < 0 || tolerance < 0 || tolerance > 0xffff || (entry & 0xf) > URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE) return URH_ERR_INVALID;
    if (!(entry & URH_STREAM_RESIDENT) && (ring < 2 || ring > URH_STREAM_MAX_RING)) return URH_ERR_INVALID;
    if ((entry & 0xf) != URH_STREAM_ENTRY_GRAB_PULSE_LENS && urh_iq_bytes(dtype) == 0) return URH_ERR_DTYPE;
    if ((entry & URH_STREAM_PSK) && (entry & 0xf) != URH_STREAM_ENTRY_AFP_DEMOD && (entry & 0xf) != URH_STREAM_ENTRY_DEMOD_DIGITIZE)
        return URH_ERR_INVALID;
    const StreamSizes z = stream_sizes(n, dtype, tolerance, chunk_samples, ring, entry);
    const bool digitize = (entry & 0xf) != URH_STREAM_ENTRY_AFP_DEMOD;
    // rows -1: the bound no capture exceeds; -2: what the resident finish reserves up front (finish.cu: n / 64 + 1024)
    const int64_t r = rows == -2 ? n / 64 + 1024 : (rows < 0 ? rows_bound(n, tolerance) : rows);
    if (entry & URH_STREAM_RESIDENT) {
        // capture + qad, full-size digitizer tables, the pulse table as urh_ensure_pulses sizes it (1.25 x rows)
        const int64_t ntiles = urh_div_up(n, URH_TILE);
        int64_t b = z.ring_bytes + ((int64_t)64 << 20);
        if (digitize)
            b += r256(ntiles * (int64_t)sizeof(UrhTileSummary)) + r256(ntiles * (int64_t)stage_cap_for(tolerance) * 4) +
                 finish_arena_bytes(ntiles, r + r / 4, true) + 16 * (r + r / 4);
        if ((entry & 0xf) == URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE)
            b += r256(ntiles * (int64_t)sizeof(UrhTileStats)) + r256((int64_t)URH_FINE_SLABS * URH_FINE_NB * 4) + r256((ntiles + 1) * 8);
        // PSK: the Costas loop's candidates, checkpoints and chain tables over the whole capture (cs_speculate)
        if (psk_order_of(entry)) b += urh_costas_arena_bytes(n, psk_order_of(entry));
        *bytes = b;
        return URH_OK;
    }
    int64_t b = z.ring_bytes;
    // the arena grows in blocks of at least 64 MiB; a request that does not fit the current block's rest opens a new one, so new
    // blocks hold at most twice the requests plus one block
    b += 2 * z.arena + ((int64_t)64 << 20);
    // look-back scan workspace (context.cu urhts::prepare): at least 8192 blocks, 256+ items each
    const int64_t nb = 2 * (z.scan_items / 256 + 1);
    b += 256 + (nb > 8192 ? nb : 8192) * (4 + 2 * 32);
    // pulse table: grown with its rows kept (old and new table alive during the copy, the new one up to twice the old)
    if (digitize) b += 3 * 16 * (r + z.rows_chunk);
    *bytes = b;
    return URH_OK;
}

extern "C" int urh_stream_stats(urh_ctx* ctx, int64_t* h_out3) {
    h_out3[0] = ctx->stream_free_low;
    h_out3[1] = ctx->stream_chunks;
    h_out3[2] = (int64_t)ctx->arena_peak;
    return URH_OK;
}

// The ring of one streamed call: the block, its events, and the copy streams drained before the block is freed on every exit path.
struct StreamRing {
    urh_ctx* ctx = nullptr;
    char* mem = nullptr;
    cudaEvent_t ev[3][URH_STREAM_MAX_RING] = {};
    int ring = 0;
    int init(urh_ctx* c, int r, int64_t bytes) {
        ctx = c;
        ring = r;
        ctx->stream_free_low = -1;
        for (int k = 0; k < 3; k++)
            for (int s = 0; s < r; s++) URH_CUDA(ctx, cudaEventCreateWithFlags(&ev[k][s], cudaEventDisableTiming));
        if (bytes > 0) URH_CUDA(ctx, cudaMallocAsync((void**)&mem, (size_t)bytes, ctx->stream));
        // the copy streams start after everything queued on the compute stream so far (the ring block included)
        URH_CUDA(ctx, cudaEventRecord(ctx->ev_comp[0], ctx->stream));
        URH_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream[0], ctx->ev_comp[0], 0));
        URH_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream[1], ctx->ev_comp[0], 0));
        return URH_OK;
    }
    ~StreamRing() {
        if (!ctx) return;
        cudaStreamSynchronize(ctx->copy_stream[0]);
        cudaStreamSynchronize(ctx->copy_stream[1]);
        if (mem) cudaFreeAsync(mem, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        for (int k = 0; k < 3; k++)
            for (int s = 0; s < ring; s++)
                if (ev[k][s]) cudaEventDestroy(ev[k][s]);
    }
};

// Runs the schedule: compute(c, s0, s1, slot) enqueues chunk c's work on the compute stream (it may synchronise).  h_src: host source
// of src_b bytes per sample uploaded into slots of src_slot bytes at d_src (NULL: the computation reads device data); h_qad: host
// destination of the qad slots at d_qad (cs floats each; NULL: none).
template <typename F>
static int stream_run(urh_ctx* ctx, int64_t n, int64_t cs, StreamRing& R, const char* h_src, int src_b, bool halo, char* d_src,
                      int64_t src_slot, float* h_qad, float* d_qad, F&& compute, bool qad_resident = false) {
    const int flags = (h_src ? URH_STREAM_UPLOAD : 0) | (h_qad ? URH_STREAM_DOWNLOAD : 0) | (halo ? URH_STREAM_HALO : 0);
    int64_t count = 0;
    URH_CHECK(urh_stream_schedule(n, cs, R.ring, flags, nullptr, 0, &count));
    std::vector<int64_t> ops((size_t)(6 * count));
    URH_CHECK(urh_stream_schedule(n, cs, R.ring, flags, ops.data(), count, &count));
    bool recorded[3][URH_STREAM_MAX_RING] = {};
    ctx->stream_chunks = 0;
    for (int64_t i = 0; i < count; i++) {
        const int64_t* o = &ops[(size_t)(6 * i)];
        const int kind = (int)o[0], s = (int)o[2];
        const int64_t c = o[1], s0 = o[3], s1 = o[4], h = o[5];
        if (kind == URH_OP_UPLOAD) {
            cudaStream_t cp = ctx->copy_stream[0];
            if (recorded[URH_OP_COMPUTE][s]) URH_CUDA(ctx, cudaStreamWaitEvent(cp, R.ev[URH_OP_COMPUTE][s], 0));
            URH_CUDA(ctx, cudaMemcpyAsync(d_src + s * src_slot + URH_STREAM_PAD - h * src_b, h_src + (s0 - h) * src_b,
                                          (size_t)((s1 - s0 + h) * src_b), cudaMemcpyHostToDevice, cp));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_UPLOAD][s], cp));
        } else if (kind == URH_OP_COMPUTE) {
            if (h_src) URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_UPLOAD][s], 0));
            if (h_qad && !qad_resident && recorded[URH_OP_DOWNLOAD][s])
                URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_DOWNLOAD][s], 0));
            URH_CHECK(compute(c, s0, s1, s));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_COMPUTE][s], ctx->stream));
            urh_stream_sample_free(ctx);
            ctx->stream_chunks++;
        } else {
            cudaStream_t cp = ctx->copy_stream[1];
            URH_CUDA(ctx, cudaStreamWaitEvent(cp, R.ev[URH_OP_COMPUTE][s], 0));
            URH_CUDA(ctx, cudaMemcpyAsync(h_qad + s0, d_qad + (qad_resident ? s0 : (int64_t)s * cs), (size_t)(s1 - s0) * sizeof(float),
                                          cudaMemcpyDeviceToHost, cp));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_DOWNLOAD][s], cp));
        }
        recorded[kind][s] = true;
    }
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream[1]));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// Per-chunk digitizer state of a streamed call: tile table and staging of one chunk, the carries between chunks, the row count.
struct StreamDigitizer {
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    UrhChain* chain;
    int cap, tol;
    bool is_ask;
    uint32_t sps;
    int64_t n, rows, rows_all;
    UrhArenaMark mark;
    int init(urh_ctx* ctx, int64_t n_total, int64_t cs, int tolerance, bool ask, uint32_t samples_per_symbol) {
        n = n_total; tol = tolerance; is_ask = ask; sps = samples_per_symbol; rows = 0;
        cap = stage_cap_for(tol);
        rows_all = rows_bound(n, tol);
        const int64_t ct = cs / URH_TILE;
        URH_CHECK(urh_arena(ctx, (size_t)ct, &tiles));
        URH_CHECK(urh_arena(ctx, (size_t)ct * cap, &staging));
        URH_CHECK(urh_arena(ctx, 8, &d_init));
        URH_CHECK(urh_arena(ctx, 1, &chain));
        URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
        mark = urh_arena_mark(ctx);
        return URH_OK;
    }
    // the chunk [s0, s1) whose dense pass has filled tiles / staging
    int finish(urh_ctx* ctx, int64_t s0, int64_t s1) {
        const int64_t rc = rows_bound(s1 - s0, tol);
        const int64_t need = rows + rc;
        if (need > (int64_t)ctx->pulses_cap_rows) {
            int64_t grow = 2 * (int64_t)ctx->pulses_cap_rows;
            if (grow > rows_all + rc) grow = rows_all + rc;
            URH_CHECK(urh_ensure_pulses_keep(ctx, (size_t)(grow > need ? grow : need), (size_t)rows));
        }
        urh_arena_release(ctx, mark);
        int64_t kc = 0;
        URH_CHECK(urh_finish_chunk(ctx, s1 - s0, tol, is_ask, sps, tiles, staging, cap, d_init, chain, s0, n, rows, rc, &kc));
        urh_stream_sample_free(ctx);
        rows += kc;
        return URH_OK;
    }
};

static int stream_check(urh_ctx* ctx, int64_t n, int ring, int mod_type, int dtype, bool iq);
// the PSK entries: the IQ is streamed, the Costas loop of chunk c continues from the state chunk c - 1 left on the device
static int psk_stream_check(urh_ctx* ctx, int64_t n, int ring, int dtype) {
    URH_CHECK(stream_check(ctx, n, ring, URH_MOD_PSK, dtype, false));
    if (n <= 2) URH_FAIL(ctx, URH_ERR_INVALID, "streamed PSK demodulation: n > 2");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    return URH_OK;
}

static int stream_check(urh_ctx* ctx, int64_t n, int ring, int mod_type, int dtype, bool iq) {
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "streamed call: empty capture");
    if (ring < 2 || ring > URH_STREAM_MAX_RING) URH_FAIL(ctx, URH_ERR_INVALID, "streamed call: ring of %d slots (2..%d)", ring, URH_STREAM_MAX_RING);
    if (iq && (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK)))
        URH_FAIL(ctx, URH_ERR_INVALID, "streamed demodulation: ASK/FSK and n > 2 (PSK is a serial recurrence)");
    if (iq && urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    return URH_OK;
}

// IQ chunk computation on slot `s`: the dense kernels over tiles [s0 / TILE, ceil(s1 / TILE)) of the whole capture.
template <bool DIG>
static int stream_dense_iq(urh_ctx* ctx, int dtype, int mod_type, const char* d_src, int64_t src_slot, int64_t n, const UrhDemodParams& dp,
                           float* qad_global, const UrhClassify& cls, int tol, StreamDigitizer* dz, int64_t s0, int64_t s1, int s,
                           UrhTileStats* ts = nullptr, const UrhFine& fine = UrhFine{}) {
    const int b = urh_iq_bytes(dtype);
    const void* iq = d_src + s * src_slot + URH_STREAM_PAD - s0 * b;   // sample i of the capture at iq + i * b for i in [s0 - 1, s1)
    const int64_t t0 = s0 / URH_TILE, t1 = urh_div_up(s1, URH_TILE);
    UrhTileSummary* tiles = dz ? dz->tiles - t0 : nullptr;
    uint32_t* staging = dz ? dz->staging - t0 * dz->cap : nullptr;
    const int cap = dz ? dz->cap : 0;
    int16_t* init = dz ? dz->d_init : nullptr;
    const int c0 = DIG ? host_classify(0.0f, cls) : 0;
    if (mod_type == URH_MOD_ASK)
        return launch_dense_iq_m<URH_MOD_ASK, DIG>(ctx, dtype, iq, n, dp, qad_global, cls, tol, tiles, staging, cap, init, c0, 0, ts, t0, t1, fine);
    return launch_dense_iq_m<URH_MOD_FSK, DIG>(ctx, dtype, iq, n, dp, qad_global, cls, tol, tiles, staging, cap, init, c0, 0, ts, t0, t1, fine);
}

// Digitizer dense pass over qad [s0, s1) at x (local view: chunk-relative tiles; only chunk 0 sets the initial state).
static int stream_dense_qad(urh_ctx* ctx, const float* x, int64_t s0, int64_t s1, const UrhClassify& cls, StreamDigitizer& dz,
                            const float* d_thr0 = nullptr, const UrhTileStats* ts = nullptr) {
    const int64_t nc = s1 - s0;
    const unsigned grid = (unsigned)urh_div_up(urh_div_up(nc, URH_TILE), URH_WARPS_PER_BLOCK);
    const int vec_in = (((uintptr_t)x % 8) == 0) ? 1 : 0;
    int16_t* init = s0 == 0 ? dz.d_init : nullptr;
    const int c0 = d_thr0 ? 0 : host_classify(0.0f, cls);
    const UrhTileStats* tsc = ts ? ts + s0 / URH_TILE : nullptr;
    if (cls.order == 2)
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, x, nc, vec_in, cls, dz.tol, dz.tiles, dz.staging,
                   dz.cap, init, c0, d_thr0, tsc);
    else
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, x, nc, vec_in, cls, dz.tol, dz.tiles, dz.staging,
                   dz.cap, init, c0, d_thr0, tsc);
    return URH_OK;
}

// ---- one-call paths: every stage enqueued on the context stream, ONE synchronisation at the end -----------------------------
struct CenterPlan;
int urh_center_chain(urh_ctx* ctx, const float* d_qad, int64_t n, const UrhTileStats* ts, int64_t max_size, int rank, int world,
                     const UrhFine* fine, CenterPlan** d_plan_out);   // center.cu
int urh_center_plan_result(urh_ctx* ctx, const CenterPlan* plan, const float** d_centerf, const double** d_center, const int** d_state);
int urh_center_plan_certify_stats(urh_ctx* ctx, const CenterPlan* plan, int64_t* h_dst3);

// Sharded demod + digitize for a KNOWN center (SURVEY 8e): dense pass over this rank's shard, then the tile-level finish with
// its three 16-byte exchanges on the stream (finish.cu).  d_qad_in != NULL: the shard is already demodulated, digitize from it.
// Every rank ends with the rows of its own shard (urh_fetch_pulses).
extern "C" int urh_shard_digitize(urh_ctx* ctx, const void* d_iq, int dtype, const float* d_qad_in, int64_t n, int has_halo,
                                  float noise_mag, int mod_type, float center, uint16_t tolerance, uint32_t samples_per_symbol,
                                  uint8_t bits_per_symbol, float center_spacing, float* d_qad_out, int64_t global_offset,
                                  int64_t n_total, int64_t* k) {
    if (!k) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "empty shard");
    if (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) URH_FAIL(ctx, URH_ERR_INVALID, "sharded path: ASK / FSK only");
    if (!d_qad_in && urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (!ctx->nccl_comm) URH_FAIL(ctx, URH_ERR_INVALID, "NCCL communicator not initialised (urh_nccl_init)");
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const int tol = tolerance;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles;
    uint32_t* staging;
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
    const int c0 = host_classify(0.0f, cls);
    if (d_qad_in) {
        const int vec_in = (((uintptr_t)d_qad_in % 8) == 0) ? 1 : 0;
        const unsigned grid = (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK);
        URH_PROF_BEGIN(ctx);
        if (cls.order == 2)
            URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad_in, n, vec_in, cls, tol, tiles, staging, cap,
                       d_init, c0, (const float*)nullptr);
        else
            URH_LAUNCH(ctx, (k_dense_f32<SrcQad, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_qad_in, n, vec_in, cls, tol, tiles, staging, cap,
                       d_init, c0, (const float*)nullptr);
        URH_PROF_END(ctx);
    } else {
        const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
        if (mod_type == URH_MOD_ASK)
            URH_CHECK((launch_dense_iq_m<URH_MOD_ASK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0, has_halo)));
        else
            URH_CHECK((launch_dense_iq_m<URH_MOD_FSK, true>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, d_init, c0, has_halo)));
    }
    return urh_finish_shard(ctx, n, tol, mod_type == URH_MOD_ASK, samples_per_symbol, tiles, staging, cap, d_init, global_offset, n_total, k);
}

// demod (ASK / FSK) + capture-wide detect_center + digitize (binary symbols) in one call (BASELINE configs[1]).
// sharded != 0: this rank's shard of a capture spread over the context's NCCL communicator (has_halo as urh_shard_dense).
// *center_state: 0 = detect_center finds no center (None; *k = 0), 1 = *center is valid, 2 = the device could not decide
// (a tie between histogram peaks whose order numpy's argsort defines, or more than 6000 bins): d_qad_out is valid, the
// caller finishes through the stepwise entry points (urh_center_window_stats / urh_center_histogram_tiles / urh_grab_pulse_lens).
// sc != NULL: the IQ is streamed from sc->h_iq through a ring (d_iq unused), qad stays resident in d_qad_out (mirrored to sc->h_qad),
// and the digitizer runs chunk by chunk over it with chained finishes, so no table grows with n but the tile statistics.
struct StreamCenter {
    int ring;
    int64_t chunk_samples;
    const void* h_iq;
    float* h_qad;
    int64_t* kept;
};
static int demod_center_digitize_impl(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag, int mod_type,
                                      uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, float* d_qad_out, bool sharded,
                                      int64_t global_offset, int64_t n_total, double* center, int* center_state, int64_t* k,
                                      const void* h_iq = nullptr, int64_t chunk_samples = 0, const StreamCenter* sc = nullptr) {
    if (!k || !center || !center_state) return URH_ERR_INVALID;
    *k = 0;
    *center = 0.0;
    *center_state = 0;
    ctx->pulses_k = 0;
    if (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) || !d_qad_out)
        URH_FAIL(ctx, URH_ERR_INVALID, "demod_center_digitize: ASK/FSK, n > 2 and a qad buffer are required");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (sharded && !ctx->nccl_comm) URH_FAIL(ctx, URH_ERR_INVALID, "NCCL communicator not initialised (urh_nccl_init)");
    urh_arena_reset(ctx);
    URH_TL_RESET(ctx);
    URH_TL_MARK(ctx, "step start");
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    UrhClassify cls;
    memset(&cls, 0, sizeof(cls));
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    UrhTileStats* ts;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &ts));
    // fine histogram of the kept samples, per slab of tiles: lets detect_center certify its peaks without a histogram pass over qad
    // (center.cu, k_center_certify).  Not collected for a sharded capture; $URH_B200_CENTER_NO_CERTIFY=1 forces the histogram pass.
    const bool no_certify = getenv("URH_B200_CENTER_NO_CERTIFY") != nullptr;   // read per call: tests compare both paths
    UrhFine fine = {};
    if (!sharded && !no_certify) {
        fine.slab_tiles = urh_div_up(ntiles, URH_FINE_SLABS);
        if (fine.slab_tiles < URH_WARPS_PER_BLOCK) fine.slab_tiles = URH_WARPS_PER_BLOCK;   // a block straddles at most one slab edge
        const int64_t nslabs = urh_div_up(ntiles, fine.slab_tiles);
        URH_CHECK(urh_arena(ctx, (size_t)(nslabs * URH_FINE_NB), &fine.gh));
        URH_CUDA(ctx, cudaMemsetAsync(fine.gh, 0, (size_t)(nslabs * URH_FINE_NB) * sizeof(unsigned int), ctx->stream));
        fine.scale = (mod_type == URH_MOD_FSK) ? 512.0f : 4096.0f;
        fine.off = (mod_type == URH_MOD_FSK) ? 2048.0f : 0.0f;
    }
    // h_iq != NULL: the capture is in (pinned) host memory.  It is uploaded in chunks on the copy stream and every chunk is
    // demodulated as soon as it has landed, so the demodulation pass hides behind the PCIe transfer.
    const int64_t chunk_tiles = (h_iq && chunk_samples > 0) ? (chunk_samples >= URH_TILE ? chunk_samples / URH_TILE : 1) : ntiles;
    const size_t sample_bytes = (size_t)urh_iq_bytes(dtype);
    StreamRing ring;
    int64_t scs = 0;
    if (sc) {
        const StreamSizes z = stream_sizes(n, dtype, tolerance, sc->chunk_samples, sc->ring, URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE);
        scs = z.cs;
        URH_CHECK(ring.init(ctx, sc->ring, sc->ring * r256(z.src_slot)));
        const int64_t slot = r256(z.src_slot);
        URH_CHECK(stream_run(ctx, n, scs, ring, (const char*)sc->h_iq, urh_iq_bytes(dtype), true, ring.mem, slot, sc->h_qad, d_qad_out,
                             [&](int64_t, int64_t s0, int64_t s1, int s) {
                                 return stream_dense_iq<false>(ctx, dtype, mod_type, ring.mem, slot, n, dp, d_qad_out, cls, 0, nullptr, s0, s1, s,
                                                               ts, fine);
                             }, true));
    }
    // the digitizer's tables, filled by the qad digitizer after the center chain, and by the speculative pass before it
    cls.noise_value = urh_noise_value(mod_type);
    cls.order = 2;
    const int tol = tolerance;
    const int cap = stage_cap_for(tol);
    UrhTileSummary* tiles = nullptr;
    uint32_t* staging = nullptr;
    int16_t* d_init = nullptr;
    if (!sc) {
        URH_CHECK(urh_arena(ctx, (size_t)ntiles, &tiles));
        URH_CHECK(urh_arena(ctx, (size_t)ntiles * cap, &staging));
        URH_CHECK(urh_arena(ctx, 8, &d_init));
    }
    // speculative digitizing (UrhSpec, DESIGN.md §4.4.1): the pass digitizes its fast tiles at a guessed threshold, the qad digitizer
    // re-reads only the tiles whose margin does not prove the classes at the detected center.  The resident single-GPU float32 FSK
    // step only; $URH_B200_NO_SPECULATE=1 turns it off, $URH_B200_SPECULATE_GUESS=<float> replaces the guess (read per call).
    const bool speculate = !sharded && !h_iq && !sc && mod_type == URH_MOD_FSK && dtype == URH_DT_F32 &&
                           getenv("URH_B200_NO_SPECULATE") == nullptr;
    UrhSpec spec = {};
    if (speculate) {
        float* tg;
        URH_CHECK(urh_arena(ctx, 1, &tg));
        URH_CHECK(urh_arena(ctx, 1, &spec.redone));
        URH_CHECK(urh_arena(ctx, (size_t)ntiles, &spec.margin));
        spec.tg = tg;
        const char* forced = getenv("URH_B200_SPECULATE_GUESS");
        URH_LAUNCH(ctx, k_speculate_guess, 1, URH_GUESS_THREADS, 0, (const float2*)d_iq, n, dp.noise_sqrd, forced ? 1 : 0,
                   forced ? strtof(forced, nullptr) : 0.0f, tg, spec.redone);
    }
    int chunk_no = 0;
    for (int64_t t0 = 0; t0 < (sc ? 0 : ntiles); t0 += chunk_tiles, chunk_no++) {
        const int64_t t1 = (t0 + chunk_tiles < ntiles) ? t0 + chunk_tiles : ntiles;
        if (h_iq) {
            const int64_t s0 = t0 * URH_TILE, s1 = (t1 * URH_TILE < n) ? t1 * URH_TILE : n;
            cudaEvent_t ev = ctx->ev_copy[chunk_no & 1];
            URH_CUDA(ctx, cudaMemcpyAsync((char*)d_iq + (size_t)s0 * sample_bytes, (const char*)h_iq + (size_t)s0 * sample_bytes,
                                          (size_t)(s1 - s0) * sample_bytes, cudaMemcpyHostToDevice, ctx->copy_stream[0]));
            URH_CUDA(ctx, cudaEventRecord(ev, ctx->copy_stream[0]));
            URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev, 0));
        }
        if (mod_type == URH_MOD_ASK)
            URH_CHECK((launch_dense_iq_m<URH_MOD_ASK, false>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, 0, nullptr, nullptr, 0, nullptr, 0, has_halo, ts, t0, t1, fine)));
        else
            URH_CHECK((launch_dense_iq_m<URH_MOD_FSK, false>(ctx, dtype, d_iq, n, dp, d_qad_out, cls, tol, tiles, staging, cap, nullptr, 0, has_halo,
                                                             ts, t0, t1, fine, speculate ? &spec : nullptr)));
    }
    CenterPlan* plan = nullptr;
    URH_CHECK(urh_center_chain(ctx, d_qad_out, n, ts, max_size, sharded ? ctx->nccl_rank : 0, sharded ? ctx->nccl_world : 1,
                               fine.gh ? &fine : nullptr, &plan));
    const float* d_centerf;
    const double* d_center;
    const int* d_state;
    urh_center_plan_result(ctx, plan, &d_centerf, &d_center, &d_state);
    // digitizer pass over qad, threshold read from device memory
    int64_t rows = 0;
    if (sc) {
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 40, d_center, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 41, d_state, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CHECK(urh_center_plan_certify_stats(ctx, plan, ctx->h_mail + 42));
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 45, (const int64_t*)ctx->center_prefix + ntiles, sizeof(int64_t), cudaMemcpyDeviceToHost,
                                      ctx->stream));
        // the chunked digitizer synchronises per chunk anyway: learn the state first and digitize only when there is a center
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        int st0 = 0;
        memcpy(&st0, ctx->h_mail + 41, sizeof(int));
        if (st0 == 1) {
            StreamDigitizer dz;
            URH_CHECK(dz.init(ctx, n, scs, tol, mod_type == URH_MOD_ASK, samples_per_symbol));
            for (int64_t s0 = 0; s0 < n; s0 += scs) {
                const int64_t s1 = s0 + scs < n ? s0 + scs : n;
                URH_CHECK(stream_dense_qad(ctx, d_qad_out + s0, s0, s1, cls, dz, d_centerf, ts));
                URH_CHECK(dz.finish(ctx, s0, s1));
            }
            rows = dz.rows;
        }
        *sc->kept = ctx->h_mail[45];
    } else {
        URH_CUDA(ctx, cudaMemsetAsync(d_init, 0, 16, ctx->stream));
        const int vec_in = (((uintptr_t)d_qad_out % 8) == 0) ? 1 : 0;
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK), URH_WARPS_PER_BLOCK * 32, 0,
                   (const float*)d_qad_out, n, vec_in, cls, tol, tiles, staging, cap, d_init, 0, d_centerf, (const UrhTileStats*)ts, spec);
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 40, d_center, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 41, d_state, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CHECK(urh_center_plan_certify_stats(ctx, plan, ctx->h_mail + 42));
        ctx->h_mail[46] = 0;
        if (speculate) URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail + 46, spec.redone, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        if (sharded)
            URH_CHECK(urh_finish_shard(ctx, n, tol, mod_type == URH_MOD_ASK, samples_per_symbol, tiles, staging, cap, d_init, global_offset, n_total, &rows));
        else
            URH_CHECK(urh_finish_local(ctx, n, tol, mod_type == URH_MOD_ASK, samples_per_symbol, tiles, staging, cap, d_init, &rows));
    }
    // the finish synchronised the stream: the two scalars have landed
    memcpy(center, ctx->h_mail + 40, sizeof(double));
    int st = 0;
    memcpy(&st, ctx->h_mail + 41, sizeof(int));
    *center_state = st;
    ctx->center_cert[0] = ctx->h_mail[42];
    ctx->center_cert[1] = fine.gh ? URH_FINE_NB : 0;
    ctx->center_cert[2] = ctx->h_mail[44];
    const int64_t redone = (spec.hi > spec.lo) ? ctx->h_mail[46] : 0;
    ctx->spec_stats[0] = spec.hi - spec.lo;
    ctx->spec_stats[1] = spec.hi - spec.lo - redone;
    ctx->spec_stats[2] = redone;
    if (st != 1) {
        ctx->pulses_k = 0;
        rows = 0;
    }
    *k = rows;
    return URH_OK;
}

extern "C" int urh_speculate_stats(urh_ctx* ctx, int64_t* h_out3) {
    for (int i = 0; i < 3; i++) h_out3[i] = ctx->spec_stats[i];
    return URH_OK;
}

extern "C" int urh_demod_center_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                         uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, float* d_qad_out,
                                         double* center, int* center_state, int64_t* k) {
    return demod_center_digitize_impl(ctx, d_iq, dtype, n, 0, noise_mag, mod_type, tolerance, samples_per_symbol, max_size, d_qad_out, false,
                                      0, n, center, center_state, k);
}

// The same step fed from HOST memory (pinned for a truly asynchronous copy): the IQ samples are uploaded into d_iq_scratch in
// chunks of `chunk_samples` on the copy stream while the compute stream demodulates the chunks that have landed (streaming
// ingest, SURVEY 8f-2).  chunk_samples <= 0: 2^24.  Works for every IQArray dtype (int8 / int16 captures move 4x / 2x fewer bytes).
extern "C" int urh_demod_center_digitize_host(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                              uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, int64_t chunk_samples,
                                              void* d_iq_scratch, float* d_qad_out, double* center, int* center_state, int64_t* k) {
    if (!h_iq || !d_iq_scratch) return URH_ERR_INVALID;
    // the copy stream must not run ahead of work already queued on the compute stream that still reads the scratch buffer
    URH_CUDA(ctx, cudaEventRecord(ctx->ev_comp[0], ctx->stream));
    URH_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream[0], ctx->ev_comp[0], 0));
    return demod_center_digitize_impl(ctx, d_iq_scratch, dtype, n, 0, noise_mag, mod_type, tolerance, samples_per_symbol, max_size, d_qad_out,
                                      false, 0, n, center, center_state, k, h_iq, chunk_samples > 0 ? chunk_samples : ((int64_t)1 << 24));
}

// ... and for one shard of a sharded capture (the halo sample, if any, must already sit at d_iq_scratch[-1])
extern "C" int urh_shard_demod_center_digitize_host(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, int has_halo, float noise_mag,
                                                    int mod_type, uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size,
                                                    int64_t chunk_samples, void* d_iq_scratch, float* d_qad_out, int64_t global_offset,
                                                    int64_t n_total, double* center, int* center_state, int64_t* k) {
    if (!h_iq || !d_iq_scratch) return URH_ERR_INVALID;
    URH_CUDA(ctx, cudaEventRecord(ctx->ev_comp[0], ctx->stream));
    URH_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream[0], ctx->ev_comp[0], 0));
    return demod_center_digitize_impl(ctx, d_iq_scratch, dtype, n, has_halo, noise_mag, mod_type, tolerance, samples_per_symbol, max_size,
                                      d_qad_out, true, global_offset, n_total, center, center_state, k, h_iq,
                                      chunk_samples > 0 ? chunk_samples : ((int64_t)1 << 24));
}

extern "C" int urh_shard_demod_center_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag,
                                               int mod_type, uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size,
                                               float* d_qad_out, int64_t global_offset, int64_t n_total, double* center,
                                               int* center_state, int64_t* k) {
    return demod_center_digitize_impl(ctx, d_iq, dtype, n, has_halo, noise_mag, mod_type, tolerance, samples_per_symbol, max_size, d_qad_out,
                                      true, global_offset, n_total, center, center_state, k);
}

// ---- streamed entry points (include/urh_b200.h) ------------------------------------------------------------------------------------
extern "C" int urh_afp_demod_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type, int64_t chunk_samples,
                                    int ring, float* h_qad) {
    if (!h_iq || !h_qad) return URH_ERR_INVALID;
    URH_CHECK(stream_check(ctx, n, ring, mod_type, dtype, true));
    urh_arena_reset(ctx);
    const StreamSizes z = stream_sizes(n, dtype, 0, chunk_samples, ring, URH_STREAM_ENTRY_AFP_DEMOD);
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    char* d_src = R.mem;
    float* d_qad = (float*)(R.mem + ring * r256(z.src_slot));
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    UrhClassify cls;
    memset(&cls, 0, sizeof(cls));
    return stream_run(ctx, n, z.cs, R, (const char*)h_iq, urh_iq_bytes(dtype), true, d_src, r256(z.src_slot), h_qad, d_qad,
                      [&](int64_t, int64_t s0, int64_t s1, int s) {
                          return stream_dense_iq<false>(ctx, dtype, mod_type, d_src, r256(z.src_slot), n, dp, d_qad + s * z.cs - s0, cls, 0,
                                                        nullptr, s0, s1, s);
                      });
}

extern "C" int urh_grab_pulse_lens_stream(urh_ctx* ctx, const float* qad, int qad_on_device, int64_t n, float center, uint16_t tolerance,
                                          int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                          int64_t chunk_samples, int ring, int64_t* k) {
    if (!k || !qad) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    URH_CHECK(stream_check(ctx, n, ring, mod_type, 0, false));
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const StreamSizes z = stream_sizes(n, 0, tolerance, chunk_samples, ring,
                                       URH_STREAM_ENTRY_GRAB_PULSE_LENS | (qad_on_device ? URH_STREAM_QAD_ON_DEVICE : 0));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    StreamDigitizer dz;
    URH_CHECK(dz.init(ctx, n, z.cs, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol));
    char* d_src = R.mem;
    URH_CHECK(stream_run(ctx, n, z.cs, R, qad_on_device ? nullptr : (const char*)qad, 4, false, d_src, r256(z.src_slot), nullptr, nullptr,
                         [&](int64_t, int64_t s0, int64_t s1, int s) {
                             const float* x = qad_on_device ? qad + s0 : (const float*)(d_src + s * r256(z.src_slot) + URH_STREAM_PAD);
                             URH_CHECK(stream_dense_qad(ctx, x, s0, s1, cls, dz));
                             return dz.finish(ctx, s0, s1);
                         }));
    *k = dz.rows;
    return URH_OK;
}

extern "C" int urh_demod_digitize_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type, float center,
                                         uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                         int64_t chunk_samples, int ring, float* h_qad_out, int64_t* k) {
    if (!k || !h_iq) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    URH_CHECK(stream_check(ctx, n, ring, mod_type, dtype, true));
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    const StreamSizes z = stream_sizes(n, dtype, tolerance, chunk_samples, ring,
                                       URH_STREAM_ENTRY_DEMOD_DIGITIZE | (h_qad_out ? URH_STREAM_QAD_OUT : 0));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    StreamDigitizer dz;
    URH_CHECK(dz.init(ctx, n, z.cs, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol));
    char* d_src = R.mem;
    float* d_qad = h_qad_out ? (float*)(R.mem + ring * r256(z.src_slot)) : nullptr;
    URH_CHECK(stream_run(ctx, n, z.cs, R, (const char*)h_iq, urh_iq_bytes(dtype), true, d_src, r256(z.src_slot), h_qad_out, d_qad,
                         [&](int64_t, int64_t s0, int64_t s1, int s) {
                             URH_CHECK(stream_dense_iq<true>(ctx, dtype, mod_type, d_src, r256(z.src_slot), n, dp,
                                                             d_qad ? d_qad + s * z.cs - s0 : nullptr, cls, tolerance, &dz, s0, s1, s));
                             return dz.finish(ctx, s0, s1);
                         }));
    *k = dz.rows;
    return URH_OK;
}

extern "C" int urh_demod_center_digitize_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type,
                                                uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, int64_t chunk_samples,
                                                int ring, float* d_qad_out, float* h_qad_out, double* center, int* center_state,
                                                int64_t* kept, int64_t* k) {
    if (!h_iq || !d_qad_out || !kept) return URH_ERR_INVALID;
    URH_CHECK(stream_check(ctx, n, ring, mod_type, dtype, true));
    StreamCenter sc;
    sc.ring = ring; sc.chunk_samples = chunk_samples; sc.h_iq = h_iq; sc.h_qad = h_qad_out; sc.kept = kept;
    return demod_center_digitize_impl(ctx, nullptr, dtype, n, 0, noise_mag, mod_type, tolerance, samples_per_symbol, max_size, d_qad_out,
                                      false, 0, n, center, center_state, k, nullptr, 0, &sc);
}

// PSK: the Costas loop per chunk (costas_spec.cu, DESIGN.md §4.3), no halo; its tables take the arena above the chunk mark.
extern "C" int urh_afp_demod_psk_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_order,
                                        float costas_loop_bandwidth, int64_t chunk_samples, int ring, float* h_qad) {
    if (!h_iq || !h_qad) return URH_ERR_INVALID;
    URH_CHECK(psk_stream_check(ctx, n, ring, dtype));
    urh_arena_reset(ctx);
    const StreamSizes z = stream_sizes(n, dtype, 0, chunk_samples, ring, URH_STREAM_ENTRY_AFP_DEMOD | psk_entry_flags(mod_order));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    const int64_t slot = r256(z.src_slot);
    char* d_src = R.mem;
    float* d_qad = (float*)(R.mem + ring * slot);
    const UrhDemodParams dp = make_demod_params(noise_mag, URH_MOD_PSK, dtype);
    UrhCostasStream cs;
    URH_CHECK(urh_costas_stream_begin(ctx, &cs));
    const UrhArenaMark mark = urh_arena_mark(ctx);
    URH_CHECK(stream_run(ctx, n, z.cs, R, (const char*)h_iq, urh_iq_bytes(dtype), false, d_src, slot, h_qad, d_qad,
                         [&](int64_t c, int64_t s0, int64_t s1, int s) {
                             urh_arena_release(ctx, mark);
                             return urh_costas_stream_chunk(ctx, &cs, c, d_src + s * slot + URH_STREAM_PAD, dtype, s1 - s0, dp.noise_sqrd,
                                                            mod_order, costas_loop_bandwidth, d_qad + s * z.cs);
                         }));
    return urh_costas_stream_end(ctx, &cs);
}

extern "C" int urh_demod_digitize_psk_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, float center,
                                             uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                             int64_t chunk_samples, int ring, float* h_qad_out, int64_t* k) {
    if (!k || !h_iq) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    URH_CHECK(psk_stream_check(ctx, n, ring, dtype));
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, URH_MOD_PSK, center, bits_per_symbol, center_spacing));
    const int mod_order = 1 << bits_per_symbol;   // as urh_demod_digitize: afp_demod(..., 1 << bits_per_symbol, 0.1)
    const UrhDemodParams dp = make_demod_params(noise_mag, URH_MOD_PSK, dtype);
    const StreamSizes z = stream_sizes(n, dtype, tolerance, chunk_samples, ring,
                                       URH_STREAM_ENTRY_DEMOD_DIGITIZE | (h_qad_out ? URH_STREAM_QAD_OUT : 0) | psk_entry_flags(mod_order));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    const int64_t slot = r256(z.src_slot);
    char* d_src = R.mem;
    float* d_qad = (float*)(R.mem + ring * slot);
    UrhCostasStream cs;
    URH_CHECK(urh_costas_stream_begin(ctx, &cs));
    StreamDigitizer dz;
    URH_CHECK(dz.init(ctx, n, z.cs, tolerance, false, samples_per_symbol));
    URH_CHECK(stream_run(ctx, n, z.cs, R, (const char*)h_iq, urh_iq_bytes(dtype), false, d_src, slot, h_qad_out, d_qad,
                         [&](int64_t c, int64_t s0, int64_t s1, int s) {
                             urh_arena_release(ctx, dz.mark);
                             float* q = d_qad + s * z.cs;
                             URH_CHECK(urh_costas_stream_chunk(ctx, &cs, c, d_src + s * slot + URH_STREAM_PAD, dtype, s1 - s0, dp.noise_sqrd,
                                                               mod_order, 0.1f, q));
                             URH_CHECK(stream_dense_qad(ctx, q, s0, s1, cls, dz));
                             return dz.finish(ctx, s0, s1);
                         }));
    *k = dz.rows;
    return urh_costas_stream_end(ctx, &cs);
}

struct UrhShardState {
    UrhCandidates cand;
    UrhFireState fs;
    int16_t* d_prev;
};
static UrhShardState* shard_state(urh_ctx* ctx) {
    if (!ctx->shard_state) ctx->shard_state = calloc(1, sizeof(UrhShardState));
    return (UrhShardState*)ctx->shard_state;
}

// Step 2 on every rank, after the summaries were exchanged: carry_* describe the run that ends right before this
// shard (fold of the preceding shards' summaries; carry_valid = 0 on the first shard).  Positions are global.
// *last_cand_cls = class of the shard's last candidate (meaningful when *count > 0).
extern "C" int urh_shard_candidates(urh_ctx* ctx, int carry_valid, int carry_cls, int64_t carry_len, int64_t global_offset,
                                    int64_t* count, const int64_t** d_pos, const int16_t** d_cls, int* last_cand_cls) {
    if (!ctx->shard_tiles) URH_FAIL(ctx, URH_ERR_INVALID, "urh_shard_dense must precede urh_shard_candidates");
    UrhShardCarry in;
    in.valid = carry_valid; in.cls = carry_cls; in.len = carry_len;
    UrhShardState* S = shard_state(ctx);
    URH_CHECK(urh_collect_candidates_shard(ctx, ctx->shard_n, ctx->shard_tol, (const UrhTileSummary*)ctx->shard_tiles,
                                           (const uint32_t*)ctx->shard_staging, ctx->shard_cap, in, global_offset, &S->cand));
    *count = S->cand.count;
    if (d_pos) *d_pos = S->cand.pos;
    if (d_cls) *d_cls = S->cand.cls;
    if (last_cand_cls) {
        *last_cand_cls = 0;
        if (S->cand.count > 0) {
            int16_t v = 0;
            URH_CUDA(ctx, cudaMemcpyAsync(&v, S->cand.cls + S->cand.count - 1, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
            URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            *last_cand_cls = v;
        }
    }
    ctx->shard_tiles = nullptr;
    return URH_OK;
}

// host copies of the candidate table urh_shard_candidates left on the device
extern "C" int urh_fetch_candidates(urh_ctx* ctx, int64_t* h_pos, int16_t* h_cls, int64_t count) {
    UrhShardState* S = shard_state(ctx);
    if (count < 0 || count > S->cand.count) URH_FAIL(ctx, URH_ERR_INVALID, "fetch_candidates: count exceeds the table");
    if (count == 0) return URH_OK;
    URH_CUDA(ctx, cudaMemcpyAsync(h_pos, S->cand.pos, (size_t)count * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_cls, S->cand.cls, (size_t)count * sizeof(int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// Step 3 (distributed finish): prev_cls = class of the last candidate of the preceding shards (the digitizer's
// initial state on the first shard).  Returns the number of firings and the position of the last one (-1: none).
extern "C" int urh_shard_fire(urh_ctx* ctx, int prev_cls, int64_t* fired, int64_t* last_fired_pos) {
    UrhShardState* S = shard_state(ctx);
    URH_CHECK(urh_arena(ctx, 8, &S->d_prev));
    const int16_t v = (int16_t)prev_cls;
    URH_CUDA(ctx, cudaMemcpyAsync(S->d_prev, &v, sizeof(v), cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    URH_CHECK(urh_fire_stage(ctx, S->cand, S->d_prev, &S->fs, last_fired_pos));
    *fired = S->fs.F;
    return URH_OK;
}

// Step 4: this shard's rows (merged locally; equal states across a shard edge are merged by the consumer).
// prev_fired_pos = position of the last firing in the preceding shards (-1: none); emit_tail on the last shard only.
extern "C" int urh_shard_rows(urh_ctx* ctx, int64_t n_total, uint16_t tolerance, int mod_type, uint32_t samples_per_symbol,
                              int64_t prev_fired_pos, int emit_tail, int64_t* k) {
    UrhShardState* S = shard_state(ctx);
    return urh_rows_stage(ctx, S->fs, n_total, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol, prev_fired_pos, emit_tail != 0, k);
}

// Step 3 on the gathering rank: the concatenated candidate tables of all shards -> pulse table of the whole capture.
extern "C" int urh_pulses_from_table(urh_ctx* ctx, const int64_t* d_pos, const int16_t* d_cls, int64_t count, int64_t n_total,
                                     uint16_t tolerance, int mod_type, uint32_t samples_per_symbol, int init_cls, int64_t* k) {
    urh_arena_reset(ctx);
    int16_t* d_init;
    URH_CHECK(urh_arena(ctx, 8, &d_init));
    const int16_t v = (int16_t)init_cls;
    URH_CUDA(ctx, cudaMemcpyAsync(d_init, &v, sizeof(v), cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    UrhCandidates cand;
    cand.count = count;
    cand.pos = (int64_t*)d_pos;
    cand.cls = (int16_t*)d_cls;
    cand.last_cls = 0;
    cand.last_len = 0;
    return urh_pulses_from_candidates(ctx, n_total, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol, cand, d_init, k);
}

extern "C" int urh_fetch_pulses(urh_ctx* ctx, int64_t* h_rows, int64_t k) {
    if (k < 0 || k > ctx->pulses_k) URH_FAIL(ctx, URH_ERR_INVALID, "fetch_pulses: k=%lld exceeds last result %lld", (long long)k, (long long)ctx->pulses_k);
    if (k == 0) return URH_OK;
    URH_CUDA(ctx, cudaMemcpyAsync(h_rows, ctx->pulses, (size_t)k * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

extern "C" int urh_pulses_device_ptr(urh_ctx* ctx, const int64_t** d_rows, int64_t* k) {
    if (d_rows) *d_rows = ctx->pulses;
    if (k) *k = ctx->pulses_k;
    return URH_OK;
}


// ---- diagnostic: packed-division self test (tests/test_gpu_packed_div.py) ---------------------------
__global__ void k_selftest_div(uint64_t seed, int64_t count, unsigned long long* mismatches, unsigned long long* tested) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned long long bad = 0, ok = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        uint64_t h = seed + (uint64_t)i * 0x9E3779B97F4A7C15ull;
        h = (h ^ (h >> 30)) * 0xBF58476D1CE4E5B9ull;
        h = (h ^ (h >> 27)) * 0x94D049BB133111EBull;
        h ^= h >> 31;
        uint64_t g = h * 0xD6E8FEB86659FD93ull + 0x632BE59BD9B4E019ull;
        g ^= g >> 29;
        // exponents uniformly inside the window, random mantissas; a few structured cases
        const uint32_t span = URH_DIVWIN_HI - URH_DIVWIN_LO;
        uint32_t ea = URH_DIVWIN_LO + (uint32_t)((h >> 40) % span), eb = URH_DIVWIN_LO + (uint32_t)((g >> 40) % span);
        uint32_t ma = (uint32_t)h & 0x7fffff, mb = (uint32_t)g & 0x7fffff;
        if ((i & 15) == 1) ma = 0;
        if ((i & 15) == 2) mb = 0;
        if ((i & 15) == 3) { ma = 0x7fffff; }
        if ((i & 15) == 4) { mb = 0x7fffff; }
        if ((i & 15) == 5) { eb = ea; }
        float a0 = __uint_as_float((ea << 23) | ma), b0 = __uint_as_float((eb << 23) | mb);
        float a1 = __uint_as_float(((URH_DIVWIN_LO + (uint32_t)((g >> 12) % span)) << 23) | ((uint32_t)(h >> 9) & 0x7fffff));
        float b1 = __uint_as_float(((URH_DIVWIN_LO + (uint32_t)((h >> 12) % span)) << 23) | ((uint32_t)(g >> 9) & 0x7fffff));
        if ((i & 15) == 6) { a1 = __uint_as_float((URH_DIVWIN_LO << 23)); b1 = __uint_as_float(((URH_DIVWIN_HI - 1) << 23) | 0x7fffff); }
        if ((i & 15) == 8) { b1 = __uint_as_float((URH_DIVWIN_LO << 23)); a1 = __uint_as_float(((URH_DIVWIN_HI - 1) << 23) | 0x7fffff); }
        if ((i & 63) == 7) a1 = 0.0f;
        const float2 q = urh_div2_window(make_float2(a0, a1), make_float2(b0, b1));
        const float r0 = __fdiv_rn(a0, b0), r1 = __fdiv_rn(a1, b1);
        bad += (__float_as_uint(q.x) != __float_as_uint(r0)) + (__float_as_uint(q.y) != __float_as_uint(r1));
        ok += 2;
    }
    atomicAdd(mismatches, bad);
    atomicAdd(tested, ok);
}

extern "C" int urh_selftest_packed_div(urh_ctx* ctx, uint64_t seed, int64_t count, int64_t* mismatches, int64_t* tested) {
    urh_arena_reset(ctx);
    unsigned long long* d;
    URH_CHECK(urh_arena(ctx, 2, &d));
    URH_CUDA(ctx, cudaMemsetAsync(d, 0, 16, ctx->stream));
    URH_LAUNCH(ctx, k_selftest_div, (unsigned)(ctx->sm_count * 8), 256, 0, seed, count, d, d + 1);
    int64_t h[2];
    URH_CHECK(urh_read_i64(ctx, (const int64_t*)d, 2, h));
    *mismatches = h[0];
    *tested = h[1];
    return URH_OK;
}
