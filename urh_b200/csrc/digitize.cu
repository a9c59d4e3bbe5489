// afp_demod (ASK/FSK), grab_pulse_lens and the fused demod+digitize path.
//
// Reference: src/urh/cythonext/signal_functions.pyx:333-378 (afp_demod), :392-495 (grab_pulse_lens).
// See dense.cuh for the dense pass and DESIGN.md for the run/candidate restatement of the digitizer.
#include "dense.cuh"
#include "tilescan.cuh"
#include "sparse.cuh"
#include "fsk_fast.cuh"
#include "dense_f32.cuh"
#include "stream_ring.cuh"

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
// (fsk_fast.cuh: float2-paired math, same bits as the generic kernel; the input is staged through a shared-memory FIFO).
// DIGITIZE and STATS: the speculative pass of the detect-center step; the threshold is the guess *d_thr0, margin[tile] its proof.
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
        urh_fsk_full_tile<DT, DIGITIZE, WRITE, STATS>(iq, n, tile * URH_TILE, dp, qad_out, thr0, cls_noise, rt, lane, one,
                                                      STATS ? tile_stats + tile : nullptr, fifo, DIGITIZE ? tiles + tile : nullptr, fine,
                                                      fine_on ? s_fine : nullptr, fine_on ? urh_fine_row(fine, tile, block_tile0) : nullptr,
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

// The optional parts of a dense pass over IQ (launch_dense_iq); the defaults leave each of them off.
struct DensePass {
    float* qad = nullptr;                 // the demodulated samples
    const UrhDigitizer* dz = nullptr;     // digitize into dz's tables at the classes of cls (with spec: the fast tiles at the guess)
    int has_halo = 0;                     // the sample preceding the first one is readable right before d_iq
    UrhTileStats* tile_stats = nullptr;   // per-tile statistics of the kept samples
    int64_t tile_lo = 0, tile_hi = -1;    // only tiles [tile_lo, tile_hi) (a chunk that has landed); tile_hi < 0: all tiles
    UrhFine fine = {};                    // with tile_stats: the fine histogram of the kept samples
    // float32 FSK with tile statistics and qad: the fast kernel's tiles are digitized at the guess spec->tg into dz's tables, with
    // their margins; spec->lo / hi is set to that tile range
    UrhSpec* spec = nullptr;
};

template <int DT, int MOD, bool DIG>
static int launch_dense_iq_t(urh_ctx* ctx, const void* d_iq, int64_t n, const UrhDemodParams& dp, const UrhClassify& cls,
                             const DensePass& o) {
    static const UrhDigitizer none = {};
    const UrhDigitizer& dz = o.dz ? *o.dz : none;
    int16_t* init_cls = DIG ? dz.d_init : nullptr;
    const int cls_of_zero = DIG ? host_classify(0.0f, cls) : 0;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const size_t fine_smem = o.fine.gh ? (size_t)URH_FINE_NB * sizeof(unsigned int) : 0;
    const int64_t tile_lo = o.tile_lo, tile_hi = (o.tile_hi < 0 || o.tile_hi > ntiles) ? ntiles : o.tile_hi;
    const int vec_in = iq_vec_aligned(d_iq, DT) ? 1 : 0;
    const int vec_out = (o.qad && ((uintptr_t)o.qad % 8) == 0) ? 1 : 0;
    const int threads = URH_WARPS_PER_BLOCK * 32;
    auto generic = [&](int64_t begin, int64_t end) -> int {   // tiles [begin, end) clipped to the requested range
        begin = begin < tile_lo ? tile_lo : begin;
        end = end > tile_hi ? tile_hi : end;
        const int64_t count = end - begin;
        if (count <= 0) return URH_OK;
        URH_LAUNCH(ctx, (k_dense_iq<DT, MOD, DIG>), (unsigned)urh_div_up(count, URH_WARPS_PER_BLOCK), threads, fine_smem, d_iq, n, dp,
                   o.qad, vec_in, vec_out, cls, dz.tol, dz.tiles, dz.staging, dz.cap, init_cls, cls_of_zero, begin, count, o.has_halo,
                   o.tile_stats, o.fine);
        return URH_OK;
    };
    // FSK on aligned buffers with a binary digitizer: tiles 1 .. nfull-1 take the paired fast kernel
    const int64_t nfull = n / URH_TILE;
    const bool fast = MOD == URH_MOD_FSK && vec_in && (!o.qad || vec_out) && (!DIG || cls.order == 2) && nfull > 1;
    URH_PROF_BEGIN(ctx);
    if (fast) {
        const int64_t fb = tile_lo > 1 ? tile_lo : 1, fe = tile_hi < nfull ? tile_hi : nfull;
        if (fe > fb) {
            const unsigned grid = (unsigned)urh_div_up(fe - fb, URH_WARPS_PER_BLOCK);
            bool speculated = false;
            if constexpr (DT == URH_DT_F32 && MOD == URH_MOD_FSK && !DIG) {
                if (o.spec && o.tile_stats && o.qad) {
                    URH_LAUNCH(ctx, (k_fsk_fifo<DT, true, true, true>), grid, threads, fine_smem, d_iq, n, dp, o.qad, 0.0f, dp.noise_value,
                               dz.tol, dz.tiles, dz.staging, dz.cap, fb, fe - fb, o.tile_stats, o.fine, (const float*)o.spec->tg, o.spec->margin);
                    o.spec->lo = fb;
                    o.spec->hi = fe;
                    speculated = true;
                }
            }
            if (speculated) {
            } else if (o.tile_stats && o.qad && !DIG) {
                URH_LAUNCH(ctx, (k_fsk_fifo<DT, false, true, true>), grid, threads, fine_smem, d_iq, n, dp, o.qad, cls.thr[0], cls.noise_value,
                           dz.tol, dz.tiles, dz.staging, dz.cap, fb, fe - fb, o.tile_stats, o.fine);
            } else if (o.qad) {
                URH_LAUNCH(ctx, (k_fsk_fifo<DT, DIG, true, false>), grid, threads, 0, d_iq, n, dp, o.qad, cls.thr[0], cls.noise_value, dz.tol,
                           dz.tiles, dz.staging, dz.cap, fb, fe - fb, nullptr, UrhFine{});
            } else {
                URH_LAUNCH(ctx, (k_fsk_fifo<DT, DIG, false, false>), grid, threads, 0, d_iq, n, dp, o.qad, cls.thr[0], cls.noise_value, dz.tol,
                           dz.tiles, dz.staging, dz.cap, fb, fe - fb, nullptr, UrhFine{});
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

template <int DT>
static int launch_dense_iq_dt(urh_ctx* ctx, int mod_type, const void* d_iq, int64_t n, const UrhDemodParams& dp, const UrhClassify& cls,
                              const DensePass& o) {
    const bool dig = o.dz && !o.spec;
    if (mod_type == URH_MOD_ASK)
        return dig ? launch_dense_iq_t<DT, URH_MOD_ASK, true>(ctx, d_iq, n, dp, cls, o) : launch_dense_iq_t<DT, URH_MOD_ASK, false>(ctx, d_iq, n, dp, cls, o);
    return dig ? launch_dense_iq_t<DT, URH_MOD_FSK, true>(ctx, d_iq, n, dp, cls, o) : launch_dense_iq_t<DT, URH_MOD_FSK, false>(ctx, d_iq, n, dp, cls, o);
}

// The dense pass over the ASK / FSK capture d_iq[0, n) of dtype.
static int launch_dense_iq(urh_ctx* ctx, int dtype, int mod_type, const void* d_iq, int64_t n, const UrhDemodParams& dp,
                           const UrhClassify& cls, const DensePass& o) {
    switch (dtype) {
        case URH_DT_I8: return launch_dense_iq_dt<URH_DT_I8>(ctx, mod_type, d_iq, n, dp, cls, o);
        case URH_DT_U8: return launch_dense_iq_dt<URH_DT_U8>(ctx, mod_type, d_iq, n, dp, cls, o);
        case URH_DT_I16: return launch_dense_iq_dt<URH_DT_I16>(ctx, mod_type, d_iq, n, dp, cls, o);
        case URH_DT_U16: return launch_dense_iq_dt<URH_DT_U16>(ctx, mod_type, d_iq, n, dp, cls, o);
        case URH_DT_F32: return launch_dense_iq_dt<URH_DT_F32>(ctx, mod_type, d_iq, n, dp, cls, o);
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
    return launch_dense_iq(ctx, dtype, mod_type, d_iq, n, dp, cls, DensePass{d_out});
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
    URH_CHECK(launch_dense_iq(ctx, dtype, mod_type, d_iq, n, dp, cls, DensePass{d_qad_out, nullptr, halo, ts}));
    return urh_center_tiles_begin(ctx, d_qad_out, ts, n, h_kept);
}

// Opening of every entry that builds a pulse table: no rows unless it succeeds.  args_ok: the entry's other required pointers are set.
static int pulses_begin(urh_ctx* ctx, int64_t* k, bool args_ok = true) {
    if (!k || !args_ok) return URH_ERR_INVALID;
    *k = 0;
    ctx->pulses_k = 0;
    return URH_OK;
}

// The digitizer's dense pass over the qad samples [s0, s1) at x, one warp per tile of dz's tables; binary symbols take the paired
// loads.  Only the capture's first chunk (s0 == 0) stores the initial state.  d_thr0: the threshold in device memory (then c0 is
// derived on the device); ts: the demodulator's tile statistics of the capture, whose all-NOISE tiles are not read.
static int launch_dense_qad(urh_ctx* ctx, const UrhDigitizer& dz, const float* x, int64_t s0, int64_t s1, const UrhClassify& cls,
                            const float* d_thr0 = nullptr, const UrhTileStats* ts = nullptr) {
    const int64_t n = s1 - s0;
    const unsigned grid = (unsigned)urh_div_up(urh_div_up(n, URH_TILE), URH_WARPS_PER_BLOCK);
    const int vec_in = (((uintptr_t)x % 8) == 0) ? 1 : 0;
    int16_t* init = s0 == 0 ? dz.d_init : nullptr;
    const int c0 = d_thr0 ? 0 : host_classify(0.0f, cls);
    if (ts) ts += s0 / URH_TILE;
    if (cls.order == 2)
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, x, n, vec_in, cls, dz.tol, dz.tiles, dz.staging,
                   dz.cap, init, c0, d_thr0, ts);
    else
        URH_LAUNCH(ctx, (k_dense_f32<SrcQad, float>), grid, URH_WARPS_PER_BLOCK * 32, 0, x, n, vec_in, cls, dz.tol, dz.tiles, dz.staging,
                   dz.cap, init, c0, d_thr0, ts);
    return URH_OK;
}

extern "C" int urh_grab_pulse_lens(urh_ctx* ctx, const float* d_qad, int64_t n, float center, uint16_t tolerance,
                                   int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                                   float center_spacing, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k));
    if (n < 0) URH_FAIL(ctx, URH_ERR_INVALID, "negative length");
    if (n == 0) return URH_OK;  // pyx:416-417 -> empty (0,2) table
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    UrhDigitizer dz;
    URH_CHECK(dz.init(ctx, n, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol, urh_div_up(n, URH_TILE), false));
    URH_PROF_BEGIN(ctx);
    URH_CHECK(launch_dense_qad(ctx, dz, d_qad, 0, n, cls));
    URH_PROF_END(ctx);
    return finish_tiles(ctx, dz, FinishShard::local(dz), k);
}

extern "C" int urh_demod_digitize(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_mag,
                                  int mod_type, float center, uint16_t tolerance, uint32_t samples_per_symbol,
                                  uint8_t bits_per_symbol, float center_spacing, float* d_qad_out, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k));
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
    UrhDigitizer dz;
    URH_CHECK(dz.init(ctx, n, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol, urh_div_up(n, URH_TILE), false));
    URH_CHECK(launch_dense_iq(ctx, dtype, mod_type, d_iq, n, dp, cls, DensePass{d_qad_out, &dz}));
    return finish_tiles(ctx, dz, FinishShard::local(dz), k);
}

// ---- streaming through a ring of device slots (DESIGN.md §4.11) -----------------------------------------------------------------
// A chunk is a whole number of tiles (the last one excepted; URH_FILTER_TILES), so every tile has the bounds and the arithmetic it
// has in the resident call.  IQ kernels see the slot through a pointer shifted back by the chunk's first sample: they index the capture
// globally, their tile range is the chunk's, and the halo sample (uploaded with the chunk) sits where the resident buffer holds it.
// rows one digitizer pass over n samples can produce: firings are >= tol + 1 samples apart, plus the head and the tail row
static int64_t rows_bound(int64_t n, int tol) { return n / (tol + 1) + 3; }

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
// workspace of the look-back scans (context.cu urhts::prepare) after tables of up to `items` elements: twice the blocks of the
// largest launch (256+ items each), at least 8192
static int64_t scan_workspace_bytes(int64_t items) {
    const int64_t nb = 2 * (items / 256 + 1);
    return 256 + (nb > 8192 ? nb : 8192) * (4 + 2 * (int64_t)urhts::SLOT);
}
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

// Message segmentation (stats.cu urh_segment_messages, urh_segment_messages_iq_stream): the arena of one segmenter pass over `tiles`
// tiles of magnitudes (the run table: tile table, staging; the candidate collector: heads, offsets, counts, closing run, the
// candidates, at most one per 10 samples), with a second closing-run slot to spare.  Its scans use the look-back workspace
// (scan_workspace_bytes), not the arena.
static int64_t segment_arena_bytes(int64_t tiles) {
    const int64_t cap = URH_TILE / 10 + 2, cand = tiles * URH_TILE / 10 + 3;
    return r256(tiles * (int64_t)sizeof(UrhTileSummary)) + r256(tiles * cap * 4) + 2 * r256(2 * (int64_t)sizeof(RunCarry)) +
           r256(tiles * 4) + r256(tiles * 8) + r256(32) + r256(cand * 8) + r256(cand * 2);
}
SegmentStreamSizes urh_segment_stream_sizes(int64_t n, int dtype, int64_t chunk_samples) {
    SegmentStreamSizes z;
    z.cs = stream_chunk_samples(n, chunk_samples);
    z.src_slot = r256(URH_STREAM_PAD + z.cs * urh_iq_bytes(dtype));
    z.mag_bytes = r256(z.cs * 8);
    z.arena = segment_arena_bytes(z.cs / URH_TILE);
    return z;
}

extern "C" int urh_stream_footprint(int64_t n, int dtype, int tolerance, int64_t chunk_samples, int ring, int entry, int64_t rows,
                                    int64_t* bytes) {
    if (!bytes || n < 0 || tolerance < 0 || tolerance > 0xffff || (entry & 0xf) > URH_STREAM_ENTRY_ESTIMATE) return URH_ERR_INVALID;
    if ((entry & 0xf) == URH_STREAM_ENTRY_SEGMENT_MESSAGES) {
        if (urh_iq_bytes(dtype) == 0) return URH_ERR_DTYPE;
        if (entry & URH_STREAM_RESIDENT) {   // the capture, its float64 magnitudes, urh_segment_messages' tables over all of it
            const int64_t ntiles = urh_div_up(n, URH_TILE);
            *bytes = r256(n * urh_iq_bytes(dtype)) + r256(n * 8) + segment_arena_bytes(ntiles) + URH_ARENA_BLOCK + scan_workspace_bytes(ntiles);
            return URH_OK;
        }
        if (ring < 2 || ring > URH_STREAM_MAX_RING) return URH_ERR_INVALID;
        const SegmentStreamSizes z = urh_segment_stream_sizes(n, dtype, chunk_samples);
        *bytes = ring * z.src_slot + z.mag_bytes + stream_arena_bytes(z.arena) + scan_workspace_bytes(z.cs / URH_TILE);
        return URH_OK;
    }
    if ((entry & 0xf) == URH_STREAM_ENTRY_ESTIMATE) {
        // AutoInterpretation.estimate's resident path: the capture, its float64 magnitudes, and the resident demodulation of order 2
        // (capture, qad); PSK's Costas tables make that the largest of the three modulations, so one decision up front covers them all
        if (!(entry & URH_STREAM_RESIDENT)) return URH_ERR_INVALID;
        if (urh_iq_bytes(dtype) == 0) return URH_ERR_DTYPE;
        int64_t demod = 0;
        URH_CHECK(urh_stream_footprint(n, dtype, 0, chunk_samples, ring, URH_STREAM_ENTRY_AFP_DEMOD | URH_STREAM_PSK | URH_STREAM_RESIDENT,
                                       -1, &demod));
        *bytes = r256(n * 8) + demod;
        return URH_OK;
    }
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
        int64_t b = z.ring_bytes + URH_ARENA_BLOCK;
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
    int64_t b = z.ring_bytes + stream_arena_bytes(z.arena);
    b += scan_workspace_bytes(z.scan_items);
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

// The digitizer of a streamed call: tables for one chunk, reused chunk after chunk, the carries between chunks, the row count.
struct StreamDigitizer {
    UrhDigitizer dz;
    UrhChain* chain;
    int64_t rows, rows_all;
    UrhArenaMark mark;
    int init(urh_ctx* ctx, int64_t n, int64_t cs, int tol, bool ask, uint32_t sps) {
        rows = 0;
        rows_all = rows_bound(n, tol);
        URH_CHECK(dz.init(ctx, n, tol, ask, sps, cs / URH_TILE, true));
        URH_CHECK(urh_arena(ctx, 1, &chain));
        mark = urh_arena_mark(ctx);
        return URH_OK;
    }
    // the chunk [s0, s1) whose dense pass has filled the tables
    int finish(urh_ctx* ctx, int64_t s0, int64_t s1) {
        const int64_t rc = rows_bound(s1 - s0, dz.tol);
        const int64_t need = rows + rc;
        if (need > (int64_t)ctx->pulses_cap_rows) {
            int64_t grow = 2 * (int64_t)ctx->pulses_cap_rows;
            if (grow > rows_all + rc) grow = rows_all + rc;
            URH_CHECK(urh_ensure_pulses_keep(ctx, (size_t)(grow > need ? grow : need), (size_t)rows));
        }
        urh_arena_release(ctx, mark);
        int64_t kc = 0;
        URH_CHECK(finish_tiles(ctx, dz, FinishShard::chunk(chain, s0, s1, dz.n, rows, rc), &kc));
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

// Dense pass over the IQ chunk w in the ring slot at `slot`: tiles [k0 / TILE, ceil(k1 / TILE)) of the whole capture; o.qad and
// o.tile_stats are indexed globally, o.dz's tables hold the chunk's tiles.
static int stream_dense_iq(urh_ctx* ctx, int dtype, int mod_type, const char* slot, int64_t n, const UrhDemodParams& dp,
                           const UrhClassify& cls, const UrhWindow& w, DensePass o) {
    const void* iq = slot + URH_STREAM_PAD - w.k0 * urh_iq_bytes(dtype);   // sample i of the capture at iq + i * b for i in [k0 - 1, k1)
    o.tile_lo = w.k0 / URH_TILE;
    o.tile_hi = urh_div_up(w.k1, URH_TILE);
    UrhDigitizer view;
    if (o.dz) {
        view = *o.dz;
        view.tiles -= o.tile_lo;
        view.staging -= o.tile_lo * view.cap;
        o.dz = &view;
    }
    return launch_dense_iq(ctx, dtype, mod_type, iq, n, dp, cls, o);
}

// ---- one-call paths: every stage enqueued on the context stream, ONE synchronisation at the end -----------------------------
struct CenterPlan;
int urh_center_chain(urh_ctx* ctx, const float* d_qad, int64_t n, const UrhTileStats* ts, int64_t max_size, int rank, int world,
                     const UrhFine* fine, CenterPlan** d_plan_out);   // center.cu
int urh_center_plan_result(urh_ctx* ctx, const CenterPlan* plan, const float** d_centerf, const double** d_center, const int** d_state);
int urh_center_plan_certify_stats(urh_ctx* ctx, const CenterPlan* plan, int64_t* h_dst3);

// Sharded demod + digitize for a KNOWN center (SURVEY 8e): dense pass over this rank's shard, then the tile-level finish with
// its three 16-byte exchanges on the stream (finish.cu).  d_iq points at the shard's first own sample; when has_halo != 0 the sample
// that precedes the shard in the capture is stored right before it (d_iq[-1]).  d_qad_in != NULL: the shard is already demodulated,
// digitize from it.  Every rank ends with the rows of its own shard (urh_fetch_pulses).
extern "C" int urh_shard_digitize(urh_ctx* ctx, const void* d_iq, int dtype, const float* d_qad_in, int64_t n, int has_halo,
                                  float noise_mag, int mod_type, float center, uint16_t tolerance, uint32_t samples_per_symbol,
                                  uint8_t bits_per_symbol, float center_spacing, float* d_qad_out, int64_t global_offset,
                                  int64_t n_total, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k));
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "empty shard");
    if (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) URH_FAIL(ctx, URH_ERR_INVALID, "sharded path: ASK / FSK only");
    if (!d_qad_in && urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (!ctx->nccl_comm) URH_FAIL(ctx, URH_ERR_INVALID, "NCCL communicator not initialised (urh_nccl_init)");
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    UrhDigitizer dz;
    URH_CHECK(dz.init(ctx, n, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol, urh_div_up(n, URH_TILE), true));
    if (d_qad_in) {
        URH_PROF_BEGIN(ctx);
        URH_CHECK(launch_dense_qad(ctx, dz, d_qad_in, 0, n, cls));
        URH_PROF_END(ctx);
    } else {
        const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
        URH_CHECK(launch_dense_iq(ctx, dtype, mod_type, d_iq, n, dp, cls, DensePass{d_qad_out, &dz, has_halo}));
    }
    return finish_tiles(ctx, dz, FinishShard::shard(ctx, dz, global_offset, n_total), k);
}

// ---- the detect-center step: demod (ASK / FSK) + capture-wide detect_center + digitize (binary symbols) in one call ---------------
// The step's results in the context's pinned mailbox, from its word 40 on (its first words are urh_read_i64's), typed as the
// copies that land in them.
struct CenterMail {
    double center;
    int state, pad;
    int64_t cert[3];       // urh_center_plan_certify_stats: {certified, -, straddle mass}
    int64_t kept;          // kept samples (streamed step)
    unsigned int redone;   // speculated tiles the qad digitizer re-read
};
static_assert(40 * sizeof(int64_t) + sizeof(CenterMail) <= 64 * sizeof(int64_t), "CenterMail outgrows the mailbox");

// sc: the IQ is streamed from sc->h_iq through a ring of sc->ring slots, qad mirrored to sc->h_qad, sc->kept = kept samples
struct StreamCenter {
    int ring;
    int64_t chunk_samples;
    const void* h_iq;
    float* h_qad;
    int64_t* kept;
};

// What the phases of one step share.
struct CenterStep {
    const void* d_iq;   // the resident capture, or the scratch the host capture is uploaded into (streamed: unused)
    int dtype, mod_type, has_halo;
    int64_t n, ntiles;
    float* d_qad;
    UrhDemodParams dp;
    UrhClassify cls;    // binary digitizer, threshold from device memory (the demodulation reads none of it)
    UrhTileStats* ts;
    UrhFine fine;       // fine.gh == nullptr: not collected
    bool speculate;
    UrhSpec spec;
    UrhDigitizer dz;    // the tables over the whole capture (not streamed: the chunked digitizer has its own)
};

// Set-up: tile statistics; the fine histogram of the kept samples per slab of tiles, which lets detect_center certify its peaks
// without a histogram pass over qad (center.cu, k_center_certify); the digitizer's tables; speculative digitizing (UrhSpec,
// DESIGN.md §4.4.1): the demodulation pass digitizes its fast tiles at a guessed threshold, the qad digitizer re-reads only the
// tiles whose margin does not prove the classes at the detected center.
static int center_setup(urh_ctx* ctx, CenterStep& S, bool certify, bool tables, const char* forced_guess, int tol, uint32_t sps) {
    URH_CHECK(urh_arena(ctx, (size_t)S.ntiles, &S.ts));
    if (certify) {
        S.fine.slab_tiles = urh_div_up(S.ntiles, URH_FINE_SLABS);
        if (S.fine.slab_tiles < URH_WARPS_PER_BLOCK) S.fine.slab_tiles = URH_WARPS_PER_BLOCK;   // a block straddles at most one slab edge
        const int64_t nslabs = urh_div_up(S.ntiles, S.fine.slab_tiles);
        URH_CHECK(urh_arena(ctx, (size_t)(nslabs * URH_FINE_NB), &S.fine.gh));
        URH_CUDA(ctx, cudaMemsetAsync(S.fine.gh, 0, (size_t)(nslabs * URH_FINE_NB) * sizeof(unsigned int), ctx->stream));
        S.fine.scale = (S.mod_type == URH_MOD_FSK) ? 512.0f : 4096.0f;
        S.fine.off = (S.mod_type == URH_MOD_FSK) ? 2048.0f : 0.0f;
    }
    S.cls.noise_value = urh_noise_value(S.mod_type);
    S.cls.order = 2;
    if (tables) URH_CHECK(S.dz.init(ctx, S.n, tol, S.mod_type == URH_MOD_ASK, sps, S.ntiles, false));
    if (S.speculate) {
        float* tg;
        URH_CHECK(urh_arena(ctx, 1, &tg));
        URH_CHECK(urh_arena(ctx, 1, &S.spec.redone));
        URH_CHECK(urh_arena(ctx, (size_t)S.ntiles, &S.spec.margin));
        S.spec.tg = tg;
        URH_LAUNCH(ctx, k_speculate_guess, 1, URH_GUESS_THREADS, 0, (const float2*)S.d_iq, S.n, S.dp.noise_sqrd, forced_guess ? 1 : 0,
                   forced_guess ? strtof(forced_guess, nullptr) : 0.0f, tg, S.spec.redone);
    }
    return URH_OK;
}

// Demodulation of tiles [t0, t1) of the capture at S.d_iq (speculating: the fast tiles are also digitized at the guess).
static int center_demod(urh_ctx* ctx, CenterStep& S, int64_t t0, int64_t t1) {
    DensePass o{S.d_qad, nullptr, S.has_halo, S.ts, t0, t1, S.fine};
    if (S.speculate) {
        o.dz = &S.dz;
        o.spec = &S.spec;
    }
    return launch_dense_iq(ctx, S.dtype, S.mod_type, S.d_iq, S.n, S.dp, S.cls, o);
}

// Demodulation of a capture in (pinned) host memory: it is uploaded into S.d_iq in chunks on the copy stream and every chunk is
// demodulated as soon as it has landed, so the demodulation pass hides behind the PCIe transfer.
static int center_demod_host(urh_ctx* ctx, CenterStep& S, const void* h_iq, int64_t chunk_samples) {
    const int64_t chunk_tiles = chunk_samples >= URH_TILE ? chunk_samples / URH_TILE : 1;
    const size_t sample_bytes = (size_t)urh_iq_bytes(S.dtype);
    int chunk_no = 0;
    for (int64_t t0 = 0; t0 < S.ntiles; t0 += chunk_tiles, chunk_no++) {
        const int64_t t1 = (t0 + chunk_tiles < S.ntiles) ? t0 + chunk_tiles : S.ntiles;
        const int64_t s0 = t0 * URH_TILE, s1 = (t1 * URH_TILE < S.n) ? t1 * URH_TILE : S.n;
        cudaEvent_t ev = ctx->ev_copy[chunk_no & 1];
        URH_CUDA(ctx, cudaMemcpyAsync((char*)S.d_iq + (size_t)s0 * sample_bytes, (const char*)h_iq + (size_t)s0 * sample_bytes,
                                      (size_t)(s1 - s0) * sample_bytes, cudaMemcpyHostToDevice, ctx->copy_stream[0]));
        URH_CUDA(ctx, cudaEventRecord(ev, ctx->copy_stream[0]));
        URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev, 0));
        URH_CHECK(center_demod(ctx, S, t0, t1));
    }
    return URH_OK;
}

// Demodulation of a capture streamed from host memory through the ring R: qad stays resident in S.d_qad (mirrored to sc.h_qad).
// *cs = the chunk samples of the call.
static int center_demod_ring(urh_ctx* ctx, CenterStep& S, const StreamCenter& sc, int tol, StreamRing& R, int64_t* cs) {
    const StreamSizes z = stream_sizes(S.n, S.dtype, tol, sc.chunk_samples, sc.ring, URH_STREAM_ENTRY_DEMOD_CENTER_DIGITIZE);
    *cs = z.cs;
    const int64_t slot = r256(z.src_slot);
    URH_CHECK(R.init(ctx, sc.ring, sc.ring * slot));
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, S.n, S.n, 1, 0, sc.chunk_samples, nullptr, nullptr, 0, win));
    return stream_run(ctx, win, R, (const char*)sc.h_iq, urh_iq_bytes(S.dtype), R.mem, slot, sc.h_qad != nullptr,
                      [&](int64_t, const UrhWindow& w, int s) {
                          return stream_dense_iq(ctx, S.dtype, S.mod_type, R.mem + s * slot, S.n, S.dp, S.cls, w,
                                                 DensePass{S.d_qad, nullptr, 0, S.ts, 0, -1, S.fine});
                      },
                      [&](int64_t, const UrhWindow& w, int, cudaStream_t cp) {   // from the resident qad
                          URH_CUDA(ctx, cudaMemcpyAsync(sc.h_qad + w.k0, S.d_qad + w.k0, (size_t)(w.k1 - w.k0) * sizeof(float),
                                                        cudaMemcpyDeviceToHost, cp));
                          return URH_OK;
                      },
                      place_after_pad, true);
}

// center, state and certificate of the plan -> the mailbox, on the stream
static int center_copy_results(urh_ctx* ctx, const CenterPlan* plan, CenterMail* mail) {
    const double* d_center;
    const int* d_state;
    urh_center_plan_result(ctx, plan, nullptr, &d_center, &d_state);
    URH_CUDA(ctx, cudaMemcpyAsync(&mail->center, d_center, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(&mail->state, d_state, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    return urh_center_plan_certify_stats(ctx, plan, mail->cert);
}

// Digitizer tail, resident tables: one pass over qad at the detected center (after speculation most tiles only need their margin
// checked: one resident wave of warps loops over them), the results copied, then the finish, which synchronises.
static int center_digitize_resident(urh_ctx* ctx, CenterStep& S, const CenterPlan* plan, const FinishShard& sh, CenterMail* mail,
                                    int64_t* rows) {
    const float* d_centerf;
    urh_center_plan_result(ctx, plan, &d_centerf, nullptr, nullptr);
    URH_CUDA(ctx, cudaMemsetAsync(S.dz.d_init, 0, 16, ctx->stream));
    const int vec_in = (((uintptr_t)S.d_qad % 8) == 0) ? 1 : 0;
    int64_t grid = urh_div_up(S.ntiles, URH_WARPS_PER_BLOCK);
    if (S.speculate) {
        int per_sm = 0;
        URH_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_dense_f32<SrcQad2, float>, URH_WARPS_PER_BLOCK * 32, 0));
        const int64_t resident = (int64_t)ctx->sm_count * (per_sm > 0 ? per_sm : 1);
        if (grid > resident) grid = resident;
    }
    URH_LAUNCH(ctx, (k_dense_f32<SrcQad2, float>), (unsigned)grid, URH_WARPS_PER_BLOCK * 32, 0, (const float*)S.d_qad, S.n, vec_in, S.cls,
               S.dz.tol, S.dz.tiles, S.dz.staging, S.dz.cap, S.dz.d_init, 0, d_centerf, (const UrhTileStats*)S.ts, S.spec);
    URH_CHECK(center_copy_results(ctx, plan, mail));
    mail->redone = 0u;
    if (S.speculate) URH_CUDA(ctx, cudaMemcpyAsync(&mail->redone, S.spec.redone, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    return finish_tiles(ctx, S.dz, sh, rows);
}

// Digitizer tail, streamed: the chunked digitizer synchronises per chunk anyway, so learn the state first and digitize (chunks of
// cs samples with chained finishes, so no table grows with n but the tile statistics) only when there is a center.
static int center_digitize_chunked(urh_ctx* ctx, CenterStep& S, const CenterPlan* plan, int64_t cs, int tol, uint32_t sps,
                                   CenterMail* mail, int64_t* rows) {
    URH_CHECK(center_copy_results(ctx, plan, mail));
    URH_CUDA(ctx, cudaMemcpyAsync(&mail->kept, (const int64_t*)ctx->center_prefix + S.ntiles, sizeof(int64_t), cudaMemcpyDeviceToHost,
                                  ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (mail->state != 1) return URH_OK;
    const float* d_centerf;
    urh_center_plan_result(ctx, plan, &d_centerf, nullptr, nullptr);
    StreamDigitizer sd;
    URH_CHECK(sd.init(ctx, S.n, cs, tol, S.mod_type == URH_MOD_ASK, sps));
    for (int64_t s0 = 0; s0 < S.n; s0 += cs) {
        const int64_t s1 = s0 + cs < S.n ? s0 + cs : S.n;
        URH_CHECK(launch_dense_qad(ctx, sd.dz, S.d_qad + s0, s0, s1, S.cls, d_centerf, S.ts));
        URH_CHECK(sd.finish(ctx, s0, s1));
    }
    *rows = sd.rows;
    return URH_OK;
}

// (BASELINE configs[1]) sharded: this rank's shard of a capture spread over the context's NCCL communicator (has_halo as urh_shard_digitize).
// *center_state: 0 = detect_center finds no center (None; *k = 0), 1 = *center is valid, 2 = the device could not decide
// (a tie between histogram peaks whose order numpy's argsort defines, or more than 6000 bins): d_qad_out is valid, the
// caller finishes through the stepwise entry points (urh_center_window_stats / urh_center_histogram_tiles / urh_grab_pulse_lens).
// The IQ comes from d_iq, from h_iq uploaded into d_iq in chunks of chunk_samples, or from sc (d_iq unused).
static int demod_center_digitize_impl(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int has_halo, float noise_mag, int mod_type,
                                      uint16_t tolerance, uint32_t samples_per_symbol, int64_t max_size, float* d_qad_out, bool sharded,
                                      int64_t global_offset, int64_t n_total, double* center, int* center_state, int64_t* k,
                                      const void* h_iq = nullptr, int64_t chunk_samples = 0, const StreamCenter* sc = nullptr) {
    URH_CHECK(pulses_begin(ctx, k, center && center_state));
    *center = 0.0;
    *center_state = 0;
    if (n <= 2 || (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK) || !d_qad_out)
        URH_FAIL(ctx, URH_ERR_INVALID, "demod_center_digitize: ASK/FSK, n > 2 and a qad buffer are required");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (sharded && !ctx->nccl_comm) URH_FAIL(ctx, URH_ERR_INVALID, "NCCL communicator not initialised (urh_nccl_init)");
    // the step's switches, read on every call (the tests compare the paths they select): $URH_B200_CENTER_NO_CERTIFY=1 forces the
    // histogram pass over qad, $URH_B200_NO_SPECULATE=1 turns speculation off, $URH_B200_SPECULATE_GUESS=<float> replaces the guess
    const bool no_certify = getenv("URH_B200_CENTER_NO_CERTIFY") != nullptr, no_speculate = getenv("URH_B200_NO_SPECULATE") != nullptr;
    const char* forced_guess = getenv("URH_B200_SPECULATE_GUESS");
    urh_arena_reset(ctx);
    URH_TL_RESET(ctx);
    URH_TL_MARK(ctx, "step start");
    CenterStep S = {};
    S.d_iq = d_iq; S.dtype = dtype; S.mod_type = mod_type; S.has_halo = has_halo;
    S.n = n; S.ntiles = urh_div_up(n, URH_TILE);
    S.d_qad = d_qad_out;
    S.dp = make_demod_params(noise_mag, mod_type, dtype);
    // the fine histogram is not collected for a sharded capture; speculation: the resident single-GPU float32 FSK step only
    S.speculate = !sharded && !h_iq && !sc && mod_type == URH_MOD_FSK && dtype == URH_DT_F32 && !no_speculate;
    URH_CHECK(center_setup(ctx, S, !sharded && !no_certify, !sc, forced_guess, tolerance, samples_per_symbol));

    StreamRing ring;   // (freed when the step returns)
    int64_t cs = 0;
    if (sc) URH_CHECK(center_demod_ring(ctx, S, *sc, tolerance, ring, &cs));
    else if (h_iq) URH_CHECK(center_demod_host(ctx, S, h_iq, chunk_samples));
    else URH_CHECK(center_demod(ctx, S, 0, S.ntiles));

    CenterPlan* plan = nullptr;
    URH_CHECK(urh_center_chain(ctx, d_qad_out, n, S.ts, max_size, sharded ? ctx->nccl_rank : 0, sharded ? ctx->nccl_world : 1,
                               S.fine.gh ? &S.fine : nullptr, &plan));

    CenterMail* mail = (CenterMail*)(ctx->h_mail + 40);
    int64_t rows = 0;
    if (sc)
        URH_CHECK(center_digitize_chunked(ctx, S, plan, cs, tolerance, samples_per_symbol, mail, &rows));
    else
        URH_CHECK(center_digitize_resident(ctx, S, plan, sharded ? FinishShard::shard(ctx, S.dz, global_offset, n_total) : FinishShard::local(S.dz),
                                           mail, &rows));

    // the finish or the chunked tail synchronised the stream: the results have landed
    *center = mail->center;
    *center_state = mail->state;
    if (sc) *sc->kept = mail->kept;
    ctx->center_cert[0] = mail->cert[0];
    ctx->center_cert[1] = S.fine.gh ? URH_FINE_NB : 0;
    ctx->center_cert[2] = mail->cert[2];
    const int64_t redone = (S.spec.hi > S.spec.lo) ? mail->redone : 0;
    ctx->spec_stats[0] = S.spec.hi - S.spec.lo;
    ctx->spec_stats[1] = S.spec.hi - S.spec.lo - redone;
    ctx->spec_stats[2] = redone;
    if (mail->state != 1) {
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
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 1, 0, chunk_samples, nullptr, nullptr, 0, win));
    return stream_run(ctx, win, R, (const char*)h_iq, urh_iq_bytes(dtype), d_src, r256(z.src_slot), true,
                      [&](int64_t, const UrhWindow& w, int s) {
                          return stream_dense_iq(ctx, dtype, mod_type, d_src + s * r256(z.src_slot), n, dp, cls, w,
                                                 DensePass{d_qad + s * z.cs - w.k0});
                      },
                      contiguous_download(ctx, (const char*)d_qad, z.cs * 4, (char*)h_qad, 4), place_after_pad);
}

extern "C" int urh_grab_pulse_lens_stream(urh_ctx* ctx, const float* qad, int qad_on_device, int64_t n, float center, uint16_t tolerance,
                                          int mod_type, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                          int64_t chunk_samples, int ring, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k, qad != nullptr));
    URH_CHECK(stream_check(ctx, n, ring, mod_type, 0, false));
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const StreamSizes z = stream_sizes(n, 0, tolerance, chunk_samples, ring,
                                       URH_STREAM_ENTRY_GRAB_PULSE_LENS | (qad_on_device ? URH_STREAM_QAD_ON_DEVICE : 0));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    StreamDigitizer sd;
    URH_CHECK(sd.init(ctx, n, z.cs, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol));
    char* d_src = R.mem;
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
    URH_CHECK(stream_run(ctx, win, R, qad_on_device ? nullptr : (const char*)qad, 4, d_src, r256(z.src_slot), false,
                         [&](int64_t, const UrhWindow& w, int s) {
                             const float* x = qad_on_device ? qad + w.k0 : (const float*)(d_src + s * r256(z.src_slot) + URH_STREAM_PAD);
                             URH_CHECK(launch_dense_qad(ctx, sd.dz, x, w.k0, w.k1, cls));
                             return sd.finish(ctx, w.k0, w.k1);
                         },
                         no_download, place_after_pad));
    *k = sd.rows;
    return URH_OK;
}

extern "C" int urh_demod_digitize_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, int mod_type, float center,
                                         uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                         int64_t chunk_samples, int ring, float* h_qad_out, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k, h_iq != nullptr));
    URH_CHECK(stream_check(ctx, n, ring, mod_type, dtype, true));
    urh_arena_reset(ctx);
    UrhClassify cls;
    URH_CHECK(fill_classify(ctx, &cls, mod_type, center, bits_per_symbol, center_spacing));
    const UrhDemodParams dp = make_demod_params(noise_mag, mod_type, dtype);
    const StreamSizes z = stream_sizes(n, dtype, tolerance, chunk_samples, ring,
                                       URH_STREAM_ENTRY_DEMOD_DIGITIZE | (h_qad_out ? URH_STREAM_QAD_OUT : 0));
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, z.ring_bytes));
    StreamDigitizer sd;
    URH_CHECK(sd.init(ctx, n, z.cs, tolerance, mod_type == URH_MOD_ASK, samples_per_symbol));
    char* d_src = R.mem;
    float* d_qad = h_qad_out ? (float*)(R.mem + ring * r256(z.src_slot)) : nullptr;
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 1, 0, chunk_samples, nullptr, nullptr, 0, win));
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, urh_iq_bytes(dtype), d_src, r256(z.src_slot), h_qad_out != nullptr,
                         [&](int64_t, const UrhWindow& w, int s) {
                             URH_CHECK(stream_dense_iq(ctx, dtype, mod_type, d_src + s * r256(z.src_slot), n, dp, cls, w,
                                                       DensePass{d_qad ? d_qad + s * z.cs - w.k0 : nullptr, &sd.dz}));
                             return sd.finish(ctx, w.k0, w.k1);
                         },
                         contiguous_download(ctx, (const char*)d_qad, z.cs * 4, (char*)h_qad_out, 4), place_after_pad));
    *k = sd.rows;
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
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, urh_iq_bytes(dtype), d_src, slot, true,
                         [&](int64_t c, const UrhWindow& w, int s) {
                             urh_arena_release(ctx, mark);
                             return urh_costas_stream_chunk(ctx, &cs, c, d_src + s * slot + URH_STREAM_PAD, dtype, w.k1 - w.k0, dp.noise_sqrd,
                                                            mod_order, costas_loop_bandwidth, d_qad + s * z.cs);
                         },
                         contiguous_download(ctx, (const char*)d_qad, z.cs * 4, (char*)h_qad, 4), place_after_pad));
    return urh_costas_stream_end(ctx, &cs);
}

extern "C" int urh_demod_digitize_psk_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_mag, float center,
                                             uint16_t tolerance, uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                                             int64_t chunk_samples, int ring, float* h_qad_out, int64_t* k) {
    URH_CHECK(pulses_begin(ctx, k, h_iq != nullptr));
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
    StreamDigitizer sd;
    URH_CHECK(sd.init(ctx, n, z.cs, tolerance, false, samples_per_symbol));
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, urh_iq_bytes(dtype), d_src, slot, h_qad_out != nullptr,
                         [&](int64_t c, const UrhWindow& w, int s) {
                             urh_arena_release(ctx, sd.mark);
                             float* q = d_qad + s * z.cs;
                             URH_CHECK(urh_costas_stream_chunk(ctx, &cs, c, d_src + s * slot + URH_STREAM_PAD, dtype, w.k1 - w.k0, dp.noise_sqrd,
                                                               mod_order, 0.1f, q));
                             URH_CHECK(launch_dense_qad(ctx, sd.dz, q, w.k0, w.k1, cls));
                             return sd.finish(ctx, w.k0, w.k1);
                         },
                         contiguous_download(ctx, (const char*)d_qad, z.cs * 4, (char*)h_qad_out, 4), place_after_pad));
    *k = sd.rows;
    return urh_costas_stream_end(ctx, &cs);
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
