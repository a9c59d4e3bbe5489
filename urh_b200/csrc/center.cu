// detect_center on the GPU (SURVEY §8a row a6; AutoInterpretation.detect_center, AutoInterpretation.py:226-277).
//
//   rect = x[x > -4]; rect = rect[int(0.05*len) : int(0.95*len)] (optionally [:max_size])   -- trimming by RANK among kept samples
//   bins = np.arange(min(rect), max(rect) + var(rect), var(rect)); y = np.histogram(rect, bins)   -> peak picking (host)
//
// Everything is organised around the dense pass's tiles (URH_TILE samples, one warp each):
//   1. a table of per-tile {count, min, max, sum, sumsq} of the kept samples (UrhTileStats).  The FSK/ASK demodulator
//      produces it for free in the pass that writes qad (urh_afp_demod_tiles, digitize.cu); for an array that is already
//      demodulated k_tile_stats_f32 reads it once.
//   2. rank prefix over the tile counts -> the two tiles the rank window cuts; window statistics = table entries of the
//      interior tiles + a rank-exact re-read of the (at most two) cut tiles.  No pass over the samples.
//   3. histogram: ONE pass over qad.  Bin edges become float thresholds (exact, see cen_edge_table), every thread counts
//      its currently popular bins in registers and only misses touch the shared-memory histogram.
// The window and histogram kernels read their parameters from a CenterPlan: the device-resident chain (second half) fills it on
// the device, the stepwise entries from their arguments (k_center_set).
#include "dense.cuh"
#include "tilescan.cuh"

#include <math.h>
#include <stdlib.h>

int urh_window_var_bitwise(urh_ctx* ctx, const float* d_x, int64_t n, const int64_t* d_prefix, int64_t t0, int64_t t1, int64_t r0,
                           int64_t r1, float* h_out2);   // pairwise.cu

struct CenStats {
    double sum, sumsq;
    float mn, mx;
    long long cnt;
};

// ---- 1. tile table from an already-demodulated array ------------------------------------------------------------------
__global__ void __launch_bounds__(URH_WARPS_PER_BLOCK * 32)
k_tile_stats_f32(const float* __restrict__ x, int64_t n, int64_t ntiles, UrhTileStats* __restrict__ ts) {
    const int lane = threadIdx.x & 31;
    const int64_t tile = (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK + (threadIdx.x >> 5);
    if (tile >= ntiles) return;
    const int64_t base = tile * URH_TILE;
    UrhStatAcc acc;
    acc.init();
    acc.all_noise = false;   // not tracked on this path (the sentinel depends on the modulation)
    if (base + URH_TILE <= n && (((uintptr_t)x) & 15) == 0) {
        const float4* p = (const float4*)(x + base) + lane;
        constexpr int ITERS = URH_TILE / 128;
        float4 cur[4], nxt[4];
#pragma unroll
        for (int j = 0; j < 4; j++) cur[j] = __ldg(p + j * 32);
        for (int it = 0; it < ITERS; it += 4) {
            if (it + 4 < ITERS) {
#pragma unroll
                for (int j = 0; j < 4; j++) nxt[j] = __ldg(p + (it + 4 + j) * 32);
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                acc.add(cur[j].x); acc.add(cur[j].y); acc.add(cur[j].z); acc.add(cur[j].w);
            }
#pragma unroll
            for (int j = 0; j < 4; j++) cur[j] = nxt[j];
        }
    } else {
        for (int j = lane; j < URH_TILE; j += 32)
            if (base + j < n) acc.add(x[base + j]);
    }
    acc.store(ts + tile, lane);
}

// ---- 2. rank prefix, window tiles, window statistics --------------------------------------------------------------------
struct ScanKept {
    const UrhTileStats* ts;
    int64_t* prefix;
    __device__ __forceinline__ int64_t load(int64_t t) const { return ts[t].cnt; }
    __device__ __forceinline__ void post(int64_t t, const int64_t& excl, const int64_t&) const { prefix[t] = excl; }
};
struct CenAddI64 {
    __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};

// prefix[t] = kept samples of the tiles before t, prefix[ntiles] = all of them (ntiles >= 1).  Enqueued only, no synchronisation.
static int kept_prefix(urh_ctx* ctx, const UrhTileStats* ts, int64_t ntiles, int64_t* prefix) {
    ScanKept fk;
    fk.ts = ts; fk.prefix = prefix;
    return urhts::scan<int64_t, CenAddI64, ScanKept>(ctx, ntiles, (int64_t)0, CenAddI64(), fk, prefix + ntiles);
}

// block-wide exclusive rank of each thread's first kept sample inside one tile (8 consecutive samples per thread)
#define CEN_PER (URH_TILE / 256)
__device__ __forceinline__ int64_t cen_tile_ranks(const float* __restrict__ x, int64_t n, int64_t t, int64_t tile_rank0, float (&v)[CEN_PER],
                                                  int* s_pre) {
    const int64_t base = t * URH_TILE + (int64_t)threadIdx.x * CEN_PER;
    int mine = 0;
#pragma unroll
    for (int j = 0; j < CEN_PER; j++) {
        v[j] = (base + j < n) ? x[base + j] : -5.0f;
        mine += (v[j] > -4.0f) ? 1 : 0;
    }
    s_pre[threadIdx.x] = mine;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        int add = 0;
        if (threadIdx.x >= off) add = s_pre[threadIdx.x - off];
        __syncthreads();
        s_pre[threadIdx.x] += add;
        __syncthreads();
    }
    return tile_rank0 + s_pre[threadIdx.x] - mine;
}

__device__ __forceinline__ void cen_block_fold(double sum, double sq, float mn, float mx, long long cnt, CenStats* out) {
    __shared__ double s_sum[256], s_sq[256];
    __shared__ float s_mn[256], s_mx[256];
    __shared__ long long s_cnt[256];
    __syncthreads();   // a block may fold twice (device-resident chain): the previous result has been read
    s_sum[threadIdx.x] = sum; s_sq[threadIdx.x] = sq; s_mn[threadIdx.x] = mn; s_mx[threadIdx.x] = mx; s_cnt[threadIdx.x] = cnt;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
            s_sum[threadIdx.x] += s_sum[threadIdx.x + off];
            s_sq[threadIdx.x] += s_sq[threadIdx.x + off];
            s_mn[threadIdx.x] = fminf(s_mn[threadIdx.x], s_mn[threadIdx.x + off]);
            s_mx[threadIdx.x] = fmaxf(s_mx[threadIdx.x], s_mx[threadIdx.x + off]);
            s_cnt[threadIdx.x] += s_cnt[threadIdx.x + off];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        CenStats r;
        r.sum = s_sum[0]; r.sumsq = s_sq[0]; r.mn = s_mn[0]; r.mx = s_mx[0]; r.cnt = s_cnt[0];
        *out = r;
    }
}

// Rank prefix over a tile table; leaves {x, ts, prefix, n} in ctx for the window / histogram calls.
int urh_center_tiles_begin(urh_ctx* ctx, const float* d_x, const UrhTileStats* ts, int64_t n, int64_t* h_total) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    int64_t* prefix;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles + 1, &prefix));
    URH_CHECK(kept_prefix(ctx, ts, ntiles, prefix));
    URH_CHECK(urh_read_i64(ctx, prefix + ntiles, 1, h_total));
    ctx->center_prefix = prefix;
    ctx->center_ts = ts;
    ctx->center_n = n;
    ctx->center_x = d_x;
    return URH_OK;
}

static int tiles_from_array(urh_ctx* ctx, const float* d_x, int64_t n, int64_t* h_total) {
    urh_arena_reset(ctx);
    ctx->center_prefix = nullptr;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    UrhTileStats* ts;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &ts));
    URH_LAUNCH(ctx, k_tile_stats_f32, (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK), URH_WARPS_PER_BLOCK * 32, 0, d_x, n, ntiles, ts);
    return urh_center_tiles_begin(ctx, d_x, ts, n, h_total);
}

static bool tiles_match(const urh_ctx* ctx, const float* d_x, int64_t n) {
    return ctx->center_prefix && ctx->center_n == n && ctx->center_x == (const void*)d_x;
}

// np.mean / np.var of the window [r0, r1) exactly as numpy computes them for a float32 array (pairwise.cu); needs the tile
// table of the same array in the arena.  h_out2 = {mean, var} (float32 values widened to double).
extern "C" int urh_center_window_var(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double* h_out2) {
    h_out2[0] = h_out2[1] = 0.0;
    if (!tiles_match(ctx, d_qad, n)) URH_FAIL(ctx, URH_ERR_INVALID, "the tile table of this array must precede urh_center_window_var");
    if (r1 <= r0) return URH_OK;
    float mv[2];
    URH_CHECK(urh_window_var_bitwise(ctx, d_qad, n, (const int64_t*)ctx->center_prefix, 0, urh_div_up(n, URH_TILE) - 1, r0, r1, mv));
    h_out2[0] = (double)mv[0];
    h_out2[1] = (double)mv[1];
    return URH_OK;
}

// Stage 1 of the stand-alone detect_center: h_out = {count_valid, r0, r1, min, max, mean, var} of the rank-trimmed samples.
// Leaves the tile table in the arena for urh_center_histogram on the same array.
extern "C" int urh_center_stats(urh_ctx* ctx, const float* d_x, int64_t n, int64_t max_size, double* h_out) {
    for (int i = 0; i < 7; i++) h_out[i] = 0.0;
    if (n <= 0) return URH_OK;
    int64_t total = 0;
    URH_CHECK(tiles_from_array(ctx, d_x, n, &total));
    // rect[int(0.05 * len(rect)) : int(0.95 * len(rect))]  (Python float arithmetic, truncation)
    int64_t r0 = (int64_t)(0.05 * (double)total), r1 = (int64_t)(0.95 * (double)total);
    if (max_size >= 0 && r1 - r0 > max_size) r1 = r0 + max_size;
    h_out[0] = (double)total; h_out[1] = (double)r0; h_out[2] = (double)r1;
    if (r1 <= r0) return URH_OK;
    double w[5];
    URH_CHECK(urh_center_window_stats(ctx, d_x, n, r0, r1, w));
    if (w[0] <= 0.0) return URH_OK;
    h_out[3] = w[1]; h_out[4] = w[2];
    // np.var(rect) replayed bit for bit (pairwise.cu): numpy's float32 pairwise sums, float32 deviations
    float mv[2];
    URH_CHECK(urh_window_var_bitwise(ctx, d_x, n, (const int64_t*)ctx->center_prefix, 0, urh_div_up(n, URH_TILE) - 1, r0, r1, mv));
    h_out[5] = (double)mv[0];
    h_out[6] = (double)mv[1];
    return URH_OK;
}

// ---- 3. histogram -------------------------------------------------------------------------------------------------------
// Bin edges of np.histogram as FLOAT thresholds: a float sample f satisfies f >= edge_k (double) iff f >= ru(edge_k), the
// smallest float not below the edge, so the binning needs no double arithmetic and stays exact.
// fe[0..nbins] = ru(edge k); fe[nbins+1] = rd(last edge) (np.histogram closes the last bin);
// fe[nbins+2] = the smallest float that both exceeds -4 (detect_center's filter) and reaches the first edge.

// Edge k exactly as np.arange forms it: start, start + step, then start + k * delta, one rounded product and one rounded sum (no
// FMA).  Caller-given edges hmin + k * hstep are the case edge1 = hmin + hstep, delta = hstep.  The operands are references, so a
// caller that keeps them in memory reads only the one it uses.
template <typename K>
__device__ __forceinline__ double cen_edge(K k, const double& hmin, const double& edge1, const double& delta) {
    return (k == 0) ? hmin : (k == 1 ? edge1 : __dadd_rn(hmin, __dmul_rn((double)k, delta)));
}

// The thresholds of edges k0, k0 + stride, ... <= nbins, and the counters hist[k] (and xhist[k]) of those k below nbins zeroed.
__device__ __forceinline__ void cen_edge_table(long long k0, long long stride, long long nbins, const double& hmin, const double& edge1,
                                               const double& delta, float* __restrict__ fe, unsigned long long* __restrict__ hist,
                                               unsigned long long* __restrict__ xhist) {
    for (long long k = k0; k <= nbins; k += stride) {
        const double e = cen_edge(k, hmin, edge1, delta);
        fe[k] = __double2float_ru(e);
        if (k == nbins) {
            fe[nbins + 1] = __double2float_rd(e);
            fe[nbins + 2] = fmaxf(__double2float_ru(hmin), nextafterf(-4.0f, 0.0f));
        }
        if (k < nbins) {
            hist[k] = 0ull;
            if (xhist) xhist[k] = 0ull;
        }
    }
}

// FAST: the bin guess rn((f - hmin) / hstep) in float arithmetic is off by less than half a bin (the host checks
// |edge| / hstep < 2^20), so the true bin is the guess or the one below it: one table look-up, no loop.
struct HistBins {
    const float* fe;   // thresholds (shared or global)
    float f_min, f_hi, scale, off;
    int nbins;
    __device__ __forceinline__ void load(const float* fe_, float scale_, int nbins_) {
        fe = fe_; nbins = nbins_; scale = scale_;
        f_hi = fe[nbins + 1];
        f_min = fe[nbins + 2];
        off = -fe[0] * scale;
    }
    // bin of one value, -1 when it does not count (np.histogram: half-open bins, the last one closed)
    template <bool FAST>
    __device__ __forceinline__ int bin_of(float f) const {
        const bool valid = f >= f_min && f <= f_hi;
        if (FAST) {
            const float t = fmaf(f, scale, off);
            int r = __float_as_int(t + 12582912.0f) - 0x4B400000;   // round to nearest via the 1.5 * 2^23 trick
            r = max(0, min(r, nbins));
            int k = r - ((f < fe[r]) ? 1 : 0);
            k = min(k, nbins - 1);
            return valid ? k : -1;
        }
        if (!valid) return -1;
        int k = (int)((f - fe[0]) * scale);
        k = max(0, min(k, nbins - 1));
        while (k > 0 && f < fe[k]) k--;
        while (k < nbins - 1 && f >= fe[k + 1]) k++;
        return k;
    }
};

// A demodulated capture piles its samples onto a handful of bins.  Each thread keeps four bins in registers as float
// INTERVALS [lo, hi) with a count: a sample is compared with the four intervals directly (no bin index is computed on a
// hit); only a sample that falls into none of them is binned through the table and takes over the least used entry, whose
// count goes to the histogram.
struct HistCache {
    float lo0, hi0, lo1, hi1, lo2, hi2, lo3, hi3;
    int h0, h1, h2, h3;
    unsigned c0, c1, c2, c3;
    __device__ __forceinline__ void init() {
        lo0 = lo1 = lo2 = lo3 = INFINITY;   // empty interval: nothing is >= +inf
        hi0 = hi1 = hi2 = hi3 = -INFINITY;
        h0 = h1 = h2 = h3 = 0;
        c0 = c1 = c2 = c3 = 0u;
    }
};

template <bool SMEM>
__device__ __forceinline__ void hist_bump(unsigned int* s_hist, unsigned long long* hist, int k, unsigned c) {
    if (SMEM) atomicAdd(&s_hist[k], c);
    else atomicAdd(&hist[k], (unsigned long long)c);
}

// f lies inside the histogram range but in none of the cached bins
template <bool SMEM, bool FAST>
__device__ __forceinline__ void hist_miss(HistCache& hc, const HistBins& hb, unsigned int* s_hist, unsigned long long* hist, float f) {
    const int k = hb.bin_of<FAST>(f);
    if (k < 0) return;
    // the cached interval must reproduce the validity test as well: nothing below f_min, the last bin closed at f_hi
    const float lo = fmaxf(hb.fe[k], hb.f_min);
    const float hi = (k == hb.nbins - 1) ? nextafterf(hb.f_hi, INFINITY) : hb.fe[k + 1];
    unsigned cm = hc.c0; int which = 0;
    if (hc.c1 < cm) { cm = hc.c1; which = 1; }
    if (hc.c2 < cm) { cm = hc.c2; which = 2; }
    if (hc.c3 < cm) { cm = hc.c3; which = 3; }
    const int old = which == 0 ? hc.h0 : which == 1 ? hc.h1 : which == 2 ? hc.h2 : hc.h3;
    if (cm) hist_bump<SMEM>(s_hist, hist, old, cm);
    if (which == 0) { hc.h0 = k; hc.c0 = 1u; hc.lo0 = lo; hc.hi0 = hi; }
    else if (which == 1) { hc.h1 = k; hc.c1 = 1u; hc.lo1 = lo; hc.hi1 = hi; }
    else if (which == 2) { hc.h2 = k; hc.c2 = 1u; hc.lo2 = lo; hc.hi2 = hi; }
    else { hc.h3 = k; hc.c3 = 1u; hc.lo3 = lo; hc.hi3 = hi; }
}

template <bool SMEM, bool FAST>
__device__ __forceinline__ void hist_put(HistCache& hc, const HistBins& hb, unsigned int* s_hist, unsigned long long* hist, float f,
                                         unsigned one) {
    // per entry: two compares chained into one predicate and a predicated increment, spelled out in PTX.  The kernel is bound by
    // the ALU pipe (FSETP, predicate logic), so the increments are multiply-adds by a run-time 1 - IMAD runs on the
    // FMA pipe - and the hit path tests the lower validity bound only (noise samples sit below it; a sample above the last edge
    // falls through to the miss path, which tests both bounds).  miss = not below the range and in no cached bin.
    unsigned miss;
    asm("{\n\t.reg .pred p0, p1, p2, p3, pv;\n\t"
        "setp.ge.f32 p0, %5, %6;\n\tsetp.lt.and.f32 p0, %5, %7, p0;\n\t@p0 mad.lo.u32 %0, %0, %15, %15;\n\t"
        "setp.ge.f32 p1, %5, %8;\n\tsetp.lt.and.f32 p1, %5, %9, p1;\n\t@p1 mad.lo.u32 %1, %1, %15, %15;\n\t"
        "setp.ge.f32 p2, %5, %10;\n\tsetp.lt.and.f32 p2, %5, %11, p2;\n\t@p2 mad.lo.u32 %2, %2, %15, %15;\n\t"
        "setp.ge.f32 p3, %5, %12;\n\tsetp.lt.and.f32 p3, %5, %13, p3;\n\t@p3 mad.lo.u32 %3, %3, %15, %15;\n\t"
        "or.pred p0, p0, p1;\n\tor.pred p2, p2, p3;\n\tor.pred p0, p0, p2;\n\t"
        "setp.ge.f32 pv, %5, %14;\n\t"
        "and.pred pv, pv, !p0;\n\t"
        "selp.u32 %4, 1, 0, pv;\n\t}"
        : "+r"(hc.c0), "+r"(hc.c1), "+r"(hc.c2), "+r"(hc.c3), "=r"(miss)
        : "f"(f), "f"(hc.lo0), "f"(hc.hi0), "f"(hc.lo1), "f"(hc.hi1), "f"(hc.lo2), "f"(hc.hi2), "f"(hc.lo3), "f"(hc.hi3),
          "f"(hb.f_min), "r"(one));
    if (miss) hist_miss<SMEM, FAST>(hc, hb, s_hist, hist, f);
}

template <bool SMEM>
__device__ __forceinline__ void hist_flush(HistCache& hc, unsigned int* s_hist, unsigned long long* hist) {
    if (hc.c0) hist_bump<SMEM>(s_hist, hist, hc.h0, hc.c0);
    if (hc.c1) hist_bump<SMEM>(s_hist, hist, hc.h1, hc.c1);
    if (hc.c2) hist_bump<SMEM>(s_hist, hist, hc.h2, hc.c2);
    if (hc.c3) hist_bump<SMEM>(s_hist, hist, hc.h3, hc.c3);
}

// Tiles strictly between win[0] and win[1] lie entirely inside the rank window: every kept sample counts, no rank
// bookkeeping, no prefix reads.  One warp per tile, grid-stride, eight 512-byte rows in flight per warp.
// Tiles [t_first, t_end) by blocks blk of nblk (the callers pass the window's interior: win[0] + 1 .. win[1]).
template <bool SMEM, bool FAST>
__device__ __forceinline__ void hist_interior_body(const float* __restrict__ x, int64_t n, int64_t t_first, int64_t t_end, int blk, int nblk,
                                                   const float* __restrict__ g_fe, float scale, int nbins,
                                                   unsigned long long* __restrict__ hist, int edges_in_smem,
                                                   const int64_t* __restrict__ prefix) {
    extern __shared__ unsigned int s_dyn[];
    unsigned int* s_hist = s_dyn;                               // [nbins] when SMEM
    float* s_fe = (float*)(s_dyn + (SMEM ? nbins : 0));         // [nbins + 3] when edges_in_smem
    const int lane = threadIdx.x & 31;
    if (SMEM)
        for (int b = threadIdx.x; b < nbins; b += 256) s_hist[b] = 0u;
    if (edges_in_smem)
        for (int b = threadIdx.x; b < nbins + 3; b += 256) s_fe[b] = g_fe[b];
    __syncthreads();
    HistBins hb;
    if (FAST) hb.load(s_fe, scale, nbins);   // FAST is only launched with the table in shared memory (LDS, not generic LD)
    else hb.load(edges_in_smem ? s_fe : g_fe, scale, nbins);
    HistCache hc;
    hc.init();
    const int64_t gw = (int64_t)blk * 8 + (threadIdx.x >> 5), nw = (int64_t)nblk * 8;
    const bool vec = (((uintptr_t)x) & 15) == 0;
    const unsigned one = blockDim.x >> 8;   // 1 (256 threads), but not a compile-time constant: see hist_put
    {
        for (int64_t t = t_first + gw; t < t_end; t += nw) {
            if (prefix[t + 1] == prefix[t]) continue;   // no kept sample in this tile (silence): nothing to count, nothing to read
            const int64_t base = t * URH_TILE;   // interior tiles are full tiles (t < last tile)
            if (vec) {
                const float4* p = (const float4*)(x + base) + lane;
                constexpr int ITERS = URH_TILE / 128, DEPTH = 4;   // a ring of four 512-byte rows in flight per warp
                float4 buf[DEPTH];
#pragma unroll
                for (int j = 0; j < DEPTH; j++) buf[j] = __ldg(p + j * 32);
#pragma unroll 1
                for (int it = 0; it < ITERS; it += DEPTH) {
                    const bool more = it + DEPTH < ITERS;
#pragma unroll
                    for (int j = 0; j < DEPTH; j++) {
                        const float4 v = buf[j];
                        if (more) buf[j] = __ldg(p + (it + DEPTH + j) * 32);
                        hist_put<SMEM, FAST>(hc, hb, s_hist, hist, v.x, one);
                        hist_put<SMEM, FAST>(hc, hb, s_hist, hist, v.y, one);
                        hist_put<SMEM, FAST>(hc, hb, s_hist, hist, v.z, one);
                        hist_put<SMEM, FAST>(hc, hb, s_hist, hist, v.w, one);
                    }
                }
            } else {
                for (int j = lane; j < URH_TILE; j += 32) hist_put<SMEM, FAST>(hc, hb, s_hist, hist, x[base + j], one);
            }
        }
    }
    hist_flush<SMEM>(hc, s_hist, hist);
    if (SMEM) {
        __syncthreads();
        for (int b = threadIdx.x; b < nbins; b += 256)
            if (s_hist[b]) atomicAdd(&hist[b], (unsigned long long)s_hist[b]);
    }
}

// the window's first and last tile (win[0], win[1]; one block each): rank-exact, straight to the global histogram
__device__ __forceinline__ void hist_window_ends_body(const float* __restrict__ x, int64_t n, const int64_t* __restrict__ prefix,
                                                      const int64_t* __restrict__ win, int64_t r0, int64_t r1,
                                                      const float* __restrict__ g_fe, float scale, int nbins,
                                                      unsigned long long* __restrict__ hist, unsigned long long* __restrict__ hist2 = nullptr) {
    __shared__ int s_pre[256];
    const int64_t t = win[blockIdx.x];
    if (t < 0 || (blockIdx.x == 1 && t == win[0])) return;
    HistBins hb;
    hb.load(g_fe, scale, nbins);
    float v[CEN_PER];
    int64_t rank = cen_tile_ranks(x, n, t, prefix[t], v, s_pre);
#pragma unroll
    for (int j = 0; j < CEN_PER; j++) {
        const bool kept = v[j] > -4.0f;
        const int k = hb.bin_of<false>(v[j]);
        if (k >= 0 && rank >= r0 && rank < r1) {
            atomicAdd(&hist[k], 1ull);
            if (hist2) atomicAdd(&hist2[k], 1ull);
        }
        rank += kept ? 1 : 0;
    }
}

// Stage 2 of the stand-alone detect_center.  Reuses the tile table urh_center_stats left for this array; builds it if
// the caller did something else in between.
extern "C" int urh_center_histogram(urh_ctx* ctx, const float* d_x, int64_t n, int64_t r0, int64_t r1, double hmin,
                                    double hstep, int64_t nbins, int64_t* h_hist) {
    if (nbins <= 0 || n <= 0) return URH_OK;
    if (!tiles_match(ctx, d_x, n)) {
        int64_t total = 0;
        URH_CHECK(tiles_from_array(ctx, d_x, n, &total));
    }
    return urh_center_histogram_tiles(ctx, d_x, n, r0, r1, hmin, hstep, nbins, h_hist);
}

// =============================================================================================================================
// Device-resident chain: demod tile table -> window -> bin edges -> histogram -> peak pick -> center, with no host
// round trip in between (the host reads {center, state} once, together with the digitizer's row count).  The decisions
// the stepwise API leaves to numpy on the host are restated here (AutoInterpretation.py:226-277):
//   * rank window  int(0.05 * kept) .. int(0.95 * kept)  (double product, truncation), capped by max_size
//   * np.arange(min, max + var, var): length ceil((stop - start) / step); elements start, start + step, then start + k * delta
//     with delta = (start + step) - start
//   * peak pick: a peak exceeds every neighbour within max(2, int(0.05 * nbins) + 1) bins; the two most populated peaks; center =
//     mean of their left edges.  np.argsort's order among EQUAL counts is implementation-defined, so a tie that would decide
//     which peak is taken hands the decision back to the host path (state 2), as do more than CEN_MAX_BINS bins.
// Sharded captures: the kept counts, the window partials and the histogram are exchanged with NCCL on the context stream.
// The stepwise entries (urh_center_window_stats, urh_center_histogram_tiles) run the same window and histogram kernels on a plan
// that k_center_set fills from their arguments.
// =============================================================================================================================
#define CEN_MAX_BINS 6000
#define CEN_VAR_MIN_RATIO 0x1p-14   // the double tile-sum variance stands in for numpy's only down to var = mean^2 * 2^-14

struct __align__(16) CenterPlan {
    long long total, offset;   // kept samples of the capture / of the preceding shards
    long long r0, r1;          // global rank window
    long long lr0, lr1;        // this shard's part of it (local ranks)
    long long win[4];          // window tiles (cen_window_tiles)
    CenStats local;            // this shard's window partial
    double hmin, edge1, delta;
    long long nbins;
    double center;
    float centerf;             // the digitizer's threshold
    float scale;
    int fast;
    int state;                 // 0: no center; 1: center found / histogram to be built; 2: host path must decide
    unsigned int ticket;
    int certified;             // 1: k_center_certify decided the center from the fine histogram (no histogram pass over qad)
    long long straddle;        // U - L of the two deciding bins (k_center_certify)
    long long pad;
};

// counts: this shard's kept total (world == 1) or the gathered totals of all ranks
__global__ void k_center_ranks(const int64_t* __restrict__ counts, int rank, int world, int64_t max_size, CenterPlan* __restrict__ plan) {
    long long total = 0, offset = 0;
    for (int q = 0; q < world; q++) {
        if (q < rank) offset += counts[q];
        total += counts[q];
    }
    const long long kept = counts[rank];
    long long r0 = (long long)(0.05 * (double)total), r1 = (long long)(0.95 * (double)total);
    if (max_size >= 0 && r1 - r0 > max_size) r1 = r0 + max_size;
    plan->total = total; plan->offset = offset; plan->r0 = r0; plan->r1 = r1;
    long long a = r0 - offset, b = r1 - offset;
    a = a < 0 ? 0 : (a > kept ? kept : a);
    b = b < 0 ? 0 : (b > kept ? kept : b);
    plan->lr0 = a; plan->lr1 = b;
    plan->ticket = 0u;
    plan->state = 1;
    plan->certified = 0;
    plan->straddle = 0;
}

// last tile t with prefix[t] <= r (prefix has ntiles + 1 entries, prefix[ntiles] = kept): the tile holding local rank r
__device__ __forceinline__ int64_t cen_tile_of_rank(const int64_t* __restrict__ prefix, int64_t ntiles, int64_t r) {
    int64_t lo = 0, hi = ntiles;   // invariant: prefix[lo] <= r, prefix[hi] > r  (prefix[0] = 0 <= r < kept = prefix[ntiles])
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (prefix[mid] <= r) lo = mid; else hi = mid;
    }
    return lo;
}

// Tiles of the local rank window [r0, r1): w[0] holds rank r0, w[1] rank r1 - 1 (tiles without a kept sample hold no rank);
// w[2], w[3] = those tiles again where the window cuts them (covers them only partly), else -1.  All -1 for an empty window.
__device__ __forceinline__ void cen_window_tiles(const int64_t* __restrict__ prefix, int64_t ntiles, long long r0, long long r1,
                                                 long long (&w)[4]) {
    long long w0 = -1, w1 = -1, w2 = -1, w3 = -1;
    if (r1 > r0) {
        w0 = cen_tile_of_rank(prefix, ntiles, r0);
        w1 = cen_tile_of_rank(prefix, ntiles, r1 - 1);
        const bool cov0 = prefix[w0] >= r0 && prefix[w0 + 1] <= r1;
        const bool cov1 = prefix[w1] >= r0 && prefix[w1 + 1] <= r1;
        w2 = cov0 ? -1 : w0;
        w3 = (cov1 || w1 == w0) ? -1 : w1;
    }
    w[0] = w0; w[1] = w1; w[2] = w2; w[3] = w3;
}

// window tiles + {count, min, max, sum, sumsq} of this shard's window: interior tiles from the table (grid-stride), the two
// cut tiles rank-exactly (blocks 0 and 1), folded by the last block to finish.  partial: gridDim.x + 2 entries.
__global__ void __launch_bounds__(256) k_center_window(const float* __restrict__ x, int64_t n, const UrhTileStats* __restrict__ ts,
                                                      const int64_t* __restrict__ prefix, int64_t ntiles, CenterPlan* __restrict__ plan,
                                                      CenStats* __restrict__ partial) {
    __shared__ long long s_win[4];
    __shared__ int s_pre[256];
    __shared__ bool s_last;
    const long long r0 = plan->lr0, r1 = plan->lr1;
    if (threadIdx.x == 0) {
        long long w[4];
        cen_window_tiles(prefix, ntiles, r0, r1, w);
        s_win[0] = w[0]; s_win[1] = w[1]; s_win[2] = w[2]; s_win[3] = w[3];
        if (blockIdx.x == 0) { plan->win[0] = w[0]; plan->win[1] = w[1]; plan->win[2] = w[2]; plan->win[3] = w[3]; }
    }
    __syncthreads();
    double sum = 0.0, sq = 0.0;
    float mn = INFINITY, mx = -INFINITY;
    long long cnt = 0;
    if (s_win[0] >= 0) {
        for (int64_t t = s_win[0] + (int64_t)blockIdx.x * 256 + threadIdx.x; t <= s_win[1]; t += (int64_t)gridDim.x * 256) {
            const int64_t a = prefix[t], b = prefix[t + 1];
            if (b > a && a >= r0 && b <= r1) {
                const UrhTileStats v = ts[t];
                sum += v.sum; sq += v.sumsq; mn = fminf(mn, v.mn); mx = fmaxf(mx, v.mx); cnt += v.cnt;
            }
        }
    }
    cen_block_fold(sum, sq, mn, mx, cnt, partial + blockIdx.x);
    if (blockIdx.x < 2) {
        const int64_t t = s_win[2 + blockIdx.x];
        sum = 0.0; sq = 0.0; mn = INFINITY; mx = -INFINITY; cnt = 0;
        if (t >= 0) {
            float v[CEN_PER];
            int64_t rank = cen_tile_ranks(x, n, t, prefix[t], v, s_pre);
#pragma unroll
            for (int j = 0; j < CEN_PER; j++) {
                if (v[j] > -4.0f) {
                    if (rank >= r0 && rank < r1) {
                        sum += (double)v[j];
                        sq += (double)v[j] * (double)v[j];
                        mn = fminf(mn, v[j]);
                        mx = fmaxf(mx, v[j]);
                        cnt++;
                    }
                    rank++;
                }
            }
        }
        cen_block_fold(sum, sq, mn, mx, cnt, partial + gridDim.x + blockIdx.x);
    }
    // the last block to arrive folds every partial in index order (deterministic)
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&plan->ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    sum = 0.0; sq = 0.0; mn = INFINITY; mx = -INFINITY; cnt = 0;
    for (int64_t t = threadIdx.x; t < (int64_t)gridDim.x + 2; t += 256) {
        CenStats p;   // written by other blocks: read through L2
        {
            const int4* src = (const int4*)(partial + t);
            int4 w0 = __ldcg(src), w1 = __ldcg(src + 1);
            memcpy(&p, &w0, 16);
            memcpy((char*)&p + 16, &w1, 16);
        }
        sum += p.sum; sq += p.sumsq; mn = fminf(mn, p.mn); mx = fmaxf(mx, p.mx); cnt += p.cnt;
    }
    cen_block_fold(sum, sq, mn, mx, cnt, &plan->local);
}

// Bin edges and the launch parameters of the histogram from the (rank-ordered) window partials of all shards.
// parts: world entries (world == 1: &plan->local).  fe: CEN_MAX_BINS + 3 floats; hist, xhist (optional): CEN_MAX_BINS counters
// (zeroed here).
__global__ void __launch_bounds__(256) k_center_plan(const CenStats* __restrict__ parts, int world, CenterPlan* __restrict__ plan,
                                                    float* __restrict__ fe, unsigned long long* __restrict__ hist,
                                                    unsigned long long* __restrict__ xhist) {
    __shared__ int s_state;
    __shared__ long long s_nbins;
    __shared__ double s_hmin, s_edge1, s_delta;
    if (threadIdx.x == 0) {
        double cnt = 0.0, sum = 0.0, sq = 0.0;
        float mn = INFINITY, mx = -INFINITY;
        for (int q = 0; q < world; q++) {   // rank order: every rank (and every world size's replay) folds identically
            cnt += (double)parts[q].cnt;
            mn = fminf(mn, parts[q].mn);
            mx = fmaxf(mx, parts[q].mx);
            sum = __dadd_rn(sum, parts[q].sum);
            sq = __dadd_rn(sq, parts[q].sumsq);
        }
        int state = 0;
        long long nbins = 0;
        double hmin = 0.0, edge1 = 0.0, delta = 0.0;
        if (plan->r1 > plan->r0 && cnt > 0.0) {
            const double mean = __ddiv_rn(sum, cnt);
            double ss = __dsub_rn(sq, __dmul_rn(__dmul_rn(cnt, mean), mean));
            if (ss < 0.0) ss = 0.0;
            const double var = __ddiv_rn(ss, cnt);
            const double hstep = (double)__double2float_rn(var);   // np.var of a float32 array is a float32
            hmin = (double)mn;
            const double stop = __dadd_rn((double)mx, hstep);
            // numpy's float32 mean is off by up to ~2^-19 of |mean|, so its variance moves by up to mean^2 * 2^-38: below
            // var = mean^2 * 2^-14 (and for non-finite sums) that outgrows the variance's own float32 rounding, and the host
            // path replays numpy's variance instead (CEN_VAR_MIN_RATIO, AutoInterpretation.FUSED_VAR_MIN_RATIO)
            if (!(var >= __dmul_rn(__dmul_rn(mean, mean), CEN_VAR_MIN_RATIO))) state = 2;
            else if (hstep != 0.0) {
                const double val = __ddiv_rn(__dsub_rn(stop, hmin), hstep);
                if (val == val && fabs(val) < 9.0e18) {
                    const long long len = (long long)ceil(val);
                    if (len >= 2) {
                        nbins = len - 1;
                        edge1 = __dadd_rn(hmin, hstep);
                        delta = __dsub_rn(edge1, hmin);
                        state = (nbins <= CEN_MAX_BINS && delta > 0.0) ? 1 : 2;
                    }
                }
            }
        }
        plan->hmin = hmin; plan->edge1 = edge1; plan->delta = delta; plan->nbins = nbins;
        plan->state = state;
        plan->center = 0.0; plan->centerf = 0.0f;
        if (state == 1) {
            plan->scale = (float)(1.0 / delta);
            const double edge_abs = fmax(fabs(hmin), fabs(hmin + (double)nbins * delta));
            plan->fast = (edge_abs / delta < 1048576.0) ? 1 : 0;
        }
        s_state = state; s_nbins = nbins; s_hmin = hmin; s_edge1 = edge1; s_delta = delta;
    }
    __syncthreads();
    if (s_state != 1) return;
    cen_edge_table(threadIdx.x, 256, s_nbins, s_hmin, s_edge1, s_delta, fe, hist, xhist);
}

// The histogram of the window's interior tiles (plan->win[0] + 1 .. plan->win[1]).  A caller that enqueues both FAST variants gets
// only the one matching plan->fast run.  SMEM: counts in shared memory; edges_in_smem: the edge table too (FAST needs it).
// MIN_BLOCKS per SM: 3 with the table in shared memory (every register kept, no spills), 4 with it in global memory (measured faster).
template <bool SMEM, bool FAST, int MIN_BLOCKS>
__global__ void __launch_bounds__(256, MIN_BLOCKS) k_hist_interior(const float* __restrict__ x, int64_t n, const CenterPlan* __restrict__ plan,
                                                                  const float* __restrict__ g_fe, unsigned long long* __restrict__ hist,
                                                                  const int64_t* __restrict__ prefix, int edges_in_smem) {
    if (plan->state != 1 || plan->certified || (plan->fast != 0) != FAST) return;
    hist_interior_body<SMEM, FAST>(x, n, plan->win[0] + 1, plan->win[1], blockIdx.x, gridDim.x, g_fe, plan->scale, (int)plan->nbins, hist,
                                   edges_in_smem, prefix);
}

// Slabs [*sf, *se) lie wholly among the window's interior tiles (win0, win1): their fine-histogram rows count in full.
__device__ __forceinline__ void cen_full_slabs(int64_t win0, int64_t win1, int64_t slab_tiles, int64_t* sf, int64_t* se) {
    *sf = (win0 + slab_tiles) / slab_tiles;   // first slab whose first tile is >= win0 + 1
    *se = win1 / slab_tiles;                  // slabs below it end at or before win1
}

// Blocks 0 and 1: the window's first and last tile, rank-exactly, into hist (and xhist).  With a fine histogram (xhist != NULL)
// blocks 2.. bin the interior tiles of the slabs the window covers only partly into xhist: the exact part of the certificate.
__global__ void __launch_bounds__(256) k_hist_window_ends(const float* __restrict__ x, int64_t n, const int64_t* __restrict__ prefix,
                                                         const CenterPlan* __restrict__ plan, const float* __restrict__ g_fe,
                                                         unsigned long long* __restrict__ hist, unsigned long long* __restrict__ xhist,
                                                         int64_t slab_tiles) {
    if (plan->state != 1) return;
    if (blockIdx.x < 2) {
        hist_window_ends_body(x, n, prefix, (const int64_t*)plan->win, plan->lr0, plan->lr1, g_fe, plan->scale, (int)plan->nbins, hist, xhist);
        return;
    }
    const int64_t w0 = plan->win[0], w1 = plan->win[1];
    int64_t sf, se;
    cen_full_slabs(w0, w1, slab_tiles, &sf, &se);
    int64_t a_end = w1, b_begin = w1;   // no full slab: every interior tile is counted exactly
    if (sf < se) { a_end = sf * slab_tiles; b_begin = se * slab_tiles; }
    const int blk = blockIdx.x - 2, nblk = gridDim.x - 2, nbins = (int)plan->nbins;
    const float scale = plan->scale;
    if (plan->fast) {
        hist_interior_body<true, true>(x, n, w0 + 1, a_end, blk, nblk, g_fe, scale, nbins, xhist, 1, prefix);
        hist_interior_body<true, true>(x, n, b_begin, w1, blk, nblk, g_fe, scale, nbins, xhist, 1, prefix);
    } else {
        hist_interior_body<true, false>(x, n, w0 + 1, a_end, blk, nblk, g_fe, scale, nbins, xhist, 1, prefix);
        hist_interior_body<true, false>(x, n, b_begin, w1, blk, nblk, g_fe, scale, nbins, xhist, 1, prefix);
    }
}

// left edge of bin k (k_center_pick, k_center_certify)
__device__ __forceinline__ double cen_left_edge(const CenterPlan* plan, int k) {
    return cen_edge(k, plan->hmin, plan->edge1, plan->delta);
}

// ---- the certified peak pick (DESIGN.md §4.4.1) --------------------------------------------------------------------------
// The window's count in bin k lies in [L_k, U_k]: xhist (exact) plus the fine-histogram buckets of the full slabs that lie wholly
// inside the bin (L) or touch it (U).  A bucket lies wholly on one side of a float threshold t iff bucket(t) != bucket(pred(t))
// (the bucket is monotone), so the bounds are exact.  Certified when two bins are peaks for every count vector within the bounds
// and both exceed every other bin that could be a peak: then k_center_pick would pick exactly these two, whatever the counts.
// Everything is strict, so numpy's order among equal counts never matters.  Otherwise nothing changes: the histogram pass runs.
#define CERT_THREADS 512
__global__ void __launch_bounds__(CERT_THREADS) k_center_certify(const UrhFine fine, CenterPlan* __restrict__ plan, const float* __restrict__ fe,
                                                                 const unsigned long long* __restrict__ xhist, unsigned long long* __restrict__ lo,
                                                                 unsigned long long* __restrict__ hi) {
    __shared__ unsigned long long s_ge[URH_FINE_NB + 1];   // kept window samples of the full slabs in buckets >= b
    __shared__ unsigned long long s_part[CERT_THREADS];
    __shared__ unsigned char s_flag[CEN_MAX_BINS];         // 1: certainly a peak, 2: possibly a peak
    __shared__ unsigned long long s_key[3];
    __shared__ unsigned int s_certain;
    if (plan->state != 1) return;
    const int tid = threadIdx.x;
    // bucket sums over the full slabs, then suffix sums (per thread, then across threads)
    constexpr int PER = URH_FINE_NB / CERT_THREADS;
    int64_t sf, se;
    cen_full_slabs(plan->win[0], plan->win[1], fine.slab_tiles, &sf, &se);
    unsigned long long b[PER], tot = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) {
        unsigned long long v = 0;
        for (int64_t sl = sf; sl < se; sl++) v += fine.gh[sl * URH_FINE_NB + tid * PER + j];
        b[j] = v;
        tot += v;
    }
    s_part[tid] = tot;
    if (tid < 3) s_key[tid] = 0ull;
    if (tid == 0) s_certain = 0u;
    __syncthreads();
    for (int off = 1; off < CERT_THREADS; off <<= 1) {
        const unsigned long long add = (tid + off < CERT_THREADS) ? s_part[tid + off] : 0ull;
        __syncthreads();
        s_part[tid] += add;
        __syncthreads();
    }
    unsigned long long run = (tid + 1 < CERT_THREADS) ? s_part[tid + 1] : 0ull;
#pragma unroll
    for (int j = PER - 1; j >= 0; j--) {
        run += b[j];
        s_ge[tid * PER + j] = run;
    }
    if (tid == 0) s_ge[URH_FINE_NB] = 0ull;
    __syncthreads();
    // bounds of every bin: bin k = [max(fe[k], f_min), min(fe[k+1], succ(f_hi))) (the last bin: up to succ(f_hi)), as bin_of counts
    const int nbins = (int)plan->nbins;
    const float f_hi = fe[nbins + 1], f_min = fe[nbins + 2], top = nextafterf(f_hi, INFINITY);
    auto ge = [&](float t, unsigned long long& glo, unsigned long long& ghi) {   // bounds of #(kept f >= t)
        const int bt = urh_fine_bucket(t, fine.scale, fine.off);
        const bool straddles = urh_fine_bucket(nextafterf(t, -INFINITY), fine.scale, fine.off) == bt;
        ghi = s_ge[bt];
        glo = straddles ? s_ge[bt + 1] : s_ge[bt];
    };
    for (int k = tid; k < nbins; k += CERT_THREADS) {
        const float a = fmaxf(fe[k], f_min), e = (k == nbins - 1) ? top : fminf(fe[k + 1], top);
        unsigned long long l = 0, u = 0;
        if (a < e) {
            unsigned long long alo, ahi, elo, ehi;
            ge(a, alo, ahi);
            ge(e, elo, ehi);
            l = alo > ehi ? alo - ehi : 0ull;
            u = ahi - elo;
        }
        lo[k] = xhist[k] + l;
        hi[k] = xhist[k] + u;
    }
    __syncthreads();
    int window = (int)(0.05 * (double)nbins) + 1;
    if (window < 2) window = 2;
    for (int k = tid; k < nbins; k += CERT_THREADS) {
        const unsigned long long l = lo[k], u = hi[k];
        bool certain = l > 0ull, possible = u > 0ull;
        for (int d = -(window - 1); d < window && (certain || possible); d++) {
            const int j = k + d;
            if (d == 0 || j < 0 || j >= nbins) continue;
            certain = certain && l > hi[j];
            possible = possible && u > lo[j];
        }
        s_flag[k] = certain ? 1 : (possible ? 2 : 0);
        if (certain) atomicAdd(&s_certain, 1u);
    }
    __syncthreads();
    // the two certain peaks with the largest L (key: L, then the lower index), then the largest U of any other possible peak
    for (int pass = 0; pass < 3; pass++) {
        const long long p0 = pass > 0 ? (long long)(8191 - (s_key[0] & 8191)) : -1, p1 = pass > 1 ? (long long)(8191 - (s_key[1] & 8191)) : -1;
        for (int k = tid; k < nbins; k += CERT_THREADS) {
            if (k == p0 || k == p1) continue;
            if (pass < 2 && s_flag[k] == 1) atomicMax(&s_key[pass], (lo[k] << 13) | (unsigned long long)(8191 - k));
            if (pass == 2 && s_flag[k] != 0) atomicMax(&s_key[2], hi[k]);
        }
        __syncthreads();
    }
    if (tid != 0 || s_certain < 2u) return;
    const int k1 = 8191 - (int)(s_key[0] & 8191), k2 = 8191 - (int)(s_key[1] & 8191);
    plan->straddle = (long long)((hi[k1] - lo[k1]) + (hi[k2] - lo[k2]));
    if (!(lo[k2] > s_key[2])) return;   // lo[k2] <= lo[k1]
    const double c = __ddiv_rn(__dadd_rn(cen_left_edge(plan, k1), cen_left_edge(plan, k2)), 2.0);
    plan->center = c;
    plan->centerf = __double2float_rn(c);
    plan->certified = 1;
}

// peak pick (one block).  y = hist[0..nbins)
__global__ void __launch_bounds__(256) k_center_pick(const unsigned long long* __restrict__ y, CenterPlan* __restrict__ plan) {
    __shared__ unsigned long long s_best[256];
    __shared__ int s_idx[256];
    __shared__ int s_cnt[256];
    if (plan->state != 1 || plan->certified) return;
    const int nbins = (int)plan->nbins;
    int window = (int)(0.05 * (double)nbins) + 1;
    if (window < 2) window = 2;
    // pass 1: best peak; pass 2: best peak among the others.  Ties that matter -> state 2.
    unsigned long long top_val[2] = {0ull, 0ull};
    int top_idx[2] = {-1, -1};
    int found = 0;
    bool undecided = false;
    for (int pass = 0; pass < 2 && !undecided; pass++) {
        unsigned long long best = 0ull;
        int bi = -1, ties = 0;
        for (int i = threadIdx.x; i < nbins; i += 256) {
            if (pass == 1 && i == top_idx[0]) continue;
            const unsigned long long v = y[i];
            if (v == 0ull || v < best) continue;
            bool peak = true;
            for (int d = 1; d < window && peak; d++) {
                const unsigned long long a = (i + d < nbins) ? y[i + d] : 0ull;
                const unsigned long long b = (i - d >= 0) ? y[i - d] : 0ull;
                peak = v > a && v > b;
            }
            if (!peak) continue;
            if (v > best) { best = v; bi = i; ties = 1; }
            else ties++;
        }
        s_best[threadIdx.x] = best; s_idx[threadIdx.x] = bi; s_cnt[threadIdx.x] = ties;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long b = 0ull;
            int idx = -1, t = 0;
            for (int j = 0; j < 256; j++) {
                if (s_idx[j] < 0) continue;
                if (s_best[j] > b) { b = s_best[j]; idx = s_idx[j]; t = s_cnt[j]; }
                else if (s_best[j] == b) t += s_cnt[j];
            }
            s_best[0] = b; s_idx[0] = idx; s_cnt[0] = t;
        }
        __syncthreads();
        const unsigned long long b = s_best[0];
        const int idx = s_idx[0], t = s_cnt[0];
        __syncthreads();
        if (idx < 0) break;
        if (pass == 0) {
            top_val[0] = b; top_idx[0] = idx; found = 1;
            if (t == 2) {
                // exactly two peaks share the top count: both are taken, in either order (the mean is symmetric).  Find the other.
                int other = -1;
                for (int i = threadIdx.x; i < nbins; i += 256) {
                    if (i == idx || y[i] != b) continue;
                    bool peak = true;
                    for (int d = 1; d < window && peak; d++) {
                        const unsigned long long a = (i + d < nbins) ? y[i + d] : 0ull;
                        const unsigned long long c = (i - d >= 0) ? y[i - d] : 0ull;
                        peak = b > a && b > c;
                    }
                    if (peak) other = i;
                }
                s_idx[threadIdx.x] = other;
                __syncthreads();
                if (threadIdx.x == 0) {
                    int o = -1;
                    for (int j = 0; j < 256; j++) if (s_idx[j] >= 0) o = s_idx[j];
                    s_idx[0] = o;
                }
                __syncthreads();
                top_idx[1] = s_idx[0]; top_val[1] = b; found = 2;
                __syncthreads();
                break;
            }
            if (t > 2) undecided = true;
        } else {
            if (t > 1) undecided = true;
            else { top_val[1] = b; top_idx[1] = idx; found = 2; }
        }
    }
    if (threadIdx.x != 0) return;
    if (undecided) { plan->state = 2; return; }
    if (found == 0) { plan->state = 0; return; }
    double c;
    if (found == 1) c = cen_left_edge(plan, top_idx[0]);
    else c = __ddiv_rn(__dadd_rn(cen_left_edge(plan, top_idx[0]), cen_left_edge(plan, top_idx[1])), 2.0);
    plan->center = c;
    plan->centerf = __double2float_rn(c);
    plan->state = 1;
    (void)top_val;
}

// ---- the stepwise entries on the chain's kernels ------------------------------------------------------------------------------
// The plan of a stepwise call: the caller's local window [r0, r1) and, with nbins > 0, its tiles and the caller's edges
// hmin + k * hstep (edge1 = hmin + hstep, delta = hstep) with their threshold table and zeroed counters.  The window statistics need
// no tiles here: k_center_window finds them itself.  nbins + 1 threads or more.
__global__ void __launch_bounds__(256) k_center_set(const int64_t* __restrict__ prefix, int64_t ntiles, long long r0, long long r1, double hmin,
                                                   double hstep, long long nbins, float scale, int fast, CenterPlan* __restrict__ plan,
                                                   float* __restrict__ fe, unsigned long long* __restrict__ hist) {
    const double edge1 = __dadd_rn(hmin, hstep);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        plan->lr0 = r0; plan->lr1 = r1;
        plan->ticket = 0u;
        plan->state = 1;
        plan->certified = 0;
        if (nbins > 0) {
            long long w[4];
            cen_window_tiles(prefix, ntiles, r0, r1, w);
            for (int i = 0; i < 4; i++) plan->win[i] = w[i];
            plan->hmin = hmin; plan->edge1 = edge1; plan->delta = hstep; plan->nbins = nbins;
            plan->scale = scale;
            plan->fast = fast;
        }
    }
    if (nbins > 0)
        cen_edge_table((long long)blockIdx.x * blockDim.x + threadIdx.x, (long long)gridDim.x * blockDim.x, nbins, hmin, edge1, hstep, fe, hist,
                       nullptr);
}

// {count, min, max, sum, sumsq} of the kept samples whose LOCAL rank is in [r0, r1), summed in the chain's order (k_center_window):
// interior tiles from the table, the cut tiles re-read from d_qad.  A shard passes the global window minus its rank offset
// (clamped to its own count).
extern "C" int urh_center_window_stats(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double* h_out5) {
    h_out5[0] = 0.0; h_out5[1] = INFINITY; h_out5[2] = -INFINITY; h_out5[3] = 0.0; h_out5[4] = 0.0;
    if (!tiles_match(ctx, d_qad, n)) URH_FAIL(ctx, URH_ERR_INVALID, "urh_afp_demod_tiles (same qad, same n) must precede urh_center_window_stats");
    if (r1 <= r0) return URH_OK;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int64_t* prefix = (const int64_t*)ctx->center_prefix;
    CenterPlan* plan;
    CenStats* partial;
    const int nb = ctx->sm_count * 2;
    URH_CHECK(urh_arena(ctx, 1, &plan));
    URH_CHECK(urh_arena(ctx, (size_t)nb + 2, &partial));
    URH_LAUNCH(ctx, k_center_set, 1, 1, 0, prefix, ntiles, (long long)r0, (long long)r1, 0.0, 0.0, 0LL, 0.0f, 0, plan, nullptr, nullptr);
    URH_LAUNCH(ctx, k_center_window, nb, 256, 0, d_qad, n, (const UrhTileStats*)ctx->center_ts, prefix, ntiles, plan, partial);
    CenStats st;
    URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_mail, &plan->local, sizeof(CenStats), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(&st, ctx->h_mail, sizeof(st));
    h_out5[0] = (double)st.cnt; h_out5[1] = (double)st.mn; h_out5[2] = (double)st.mx; h_out5[3] = st.sum; h_out5[4] = st.sumsq;
    return URH_OK;
}

// Counts for edges hmin + k*hstep, k = 0..nbins (np.arange) over the samples of LOCAL rank [r0, r1); needs the tile
// table of the same array (urh_afp_demod_tiles / urh_center_stats) in the arena.
extern "C" int urh_center_histogram_tiles(urh_ctx* ctx, const float* d_qad, int64_t n, int64_t r0, int64_t r1, double hmin,
                                          double hstep, int64_t nbins, int64_t* h_hist) {
    if (nbins <= 0) return URH_OK;
    if (!tiles_match(ctx, d_qad, n)) URH_FAIL(ctx, URH_ERR_INVALID, "urh_afp_demod_tiles (same qad, same n) must precede urh_center_histogram_tiles");
    if (nbins > (int64_t)1 << 30) URH_FAIL(ctx, URH_ERR_INVALID, "too many histogram bins");
    if (r1 <= r0) {
        memset(h_hist, 0, (size_t)nbins * sizeof(int64_t));
        return URH_OK;
    }
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int64_t* prefix = (const int64_t*)ctx->center_prefix;
    CenterPlan* plan;
    float* fe;
    unsigned long long* hist;
    URH_CHECK(urh_arena(ctx, 1, &plan));
    URH_CHECK(urh_arena(ctx, (size_t)nbins + 3, &fe));
    URH_CHECK(urh_arena(ctx, (size_t)nbins, &hist));
    // shared memory (48 KB without opt-in): histogram first, then the edge table if it still fits
    const bool in_smem = nbins <= 12000;
    const int edges_smem = (in_smem && nbins <= 6000) ? 1 : 0;
    const size_t dyn = (in_smem ? (size_t)nbins * 4 : 0) + (edges_smem ? (size_t)(nbins + 3) * 4 : 0);
    const float scale = (float)(1.0 / hstep);
    // one-look-up binning needs the float guess to be good to half a bin
    const double edge_abs = fmax(fabs(hmin), fabs(hmin + (double)nbins * hstep));
    const int fast = (edges_smem && hstep > 0.0 && edge_abs / hstep < 1048576.0) ? 1 : 0;
    const unsigned gs = (unsigned)min(urh_div_up(ntiles, 8), (int64_t)ctx->sm_count * 8);
    URH_LAUNCH(ctx, k_center_set, (unsigned)urh_div_up(nbins + 1, 256), 256, 0, prefix, ntiles, (long long)r0, (long long)r1, hmin, hstep,
               (long long)nbins, scale, fast, plan, fe, hist);
    const CenterPlan* cplan = plan;
    const float* cfe = fe;
    if (fast) URH_LAUNCH(ctx, (k_hist_interior<true, true, 3>), gs, 256, dyn, d_qad, n, cplan, cfe, hist, prefix, edges_smem);
    else if (edges_smem) URH_LAUNCH(ctx, (k_hist_interior<true, false, 3>), gs, 256, dyn, d_qad, n, cplan, cfe, hist, prefix, edges_smem);
    else if (in_smem) URH_LAUNCH(ctx, (k_hist_interior<true, false, 4>), gs, 256, dyn, d_qad, n, cplan, cfe, hist, prefix, edges_smem);
    else URH_LAUNCH(ctx, (k_hist_interior<false, false, 4>), gs, 256, dyn, d_qad, n, cplan, cfe, hist, prefix, edges_smem);
    URH_LAUNCH(ctx, k_hist_window_ends, 2, 256, 0, d_qad, n, prefix, cplan, cfe, hist, (unsigned long long*)nullptr, (int64_t)1);
    URH_CUDA(ctx, cudaMemcpyAsync(h_hist, hist, (size_t)nbins * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// The chain.  ts = the demodulator's tile table of d_qad (arena); *d_plan_out stays valid until the next arena reset.
// Enqueues everything on the context stream; no synchronisation.  world > 1: the context's NCCL communicator.
// fine != NULL (world == 1 only): the demodulator's fine histogram of d_qad; k_center_certify may then decide the center without
// the histogram pass over qad.
int urh_center_chain(urh_ctx* ctx, const float* d_qad, int64_t n, const UrhTileStats* ts, int64_t max_size, int rank, int world,
                     const UrhFine* fine, CenterPlan** d_plan_out) {
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    int64_t* prefix;
    CenterPlan* plan;
    CenStats* partial;
    float* fe;
    unsigned long long* hist;
    int64_t* d_counts;
    CenStats* d_parts;
    unsigned long long *xhist = nullptr, *cert_lo = nullptr, *cert_hi = nullptr;
    const int nb = ctx->sm_count * 2;
    URH_CHECK(urh_arena(ctx, (size_t)ntiles + 1, &prefix));
    URH_CHECK(urh_arena(ctx, 1, &plan));
    URH_CHECK(urh_arena(ctx, (size_t)nb + 2, &partial));
    URH_CHECK(urh_arena(ctx, (size_t)CEN_MAX_BINS + 3, &fe));
    URH_CHECK(urh_arena(ctx, (size_t)CEN_MAX_BINS, &hist));
    URH_CHECK(urh_arena(ctx, (size_t)world, &d_counts));
    URH_CHECK(urh_arena(ctx, (size_t)world, &d_parts));
    if (fine) {
        URH_CHECK(urh_arena(ctx, (size_t)CEN_MAX_BINS, &xhist));
        URH_CHECK(urh_arena(ctx, (size_t)CEN_MAX_BINS, &cert_lo));
        URH_CHECK(urh_arena(ctx, (size_t)CEN_MAX_BINS, &cert_hi));
    }
    URH_CHECK(kept_prefix(ctx, ts, ntiles, prefix));
    const int64_t* counts = prefix + ntiles;
    if (world > 1) {
        URH_TL_MARK(ctx, "x1 kept counts: enter");
        URH_CHECK(urh_nccl_allgather(ctx, prefix + ntiles, d_counts, sizeof(int64_t)));
        URH_TL_MARK(ctx, "x1 kept counts: done");
        counts = d_counts;
    }
    URH_LAUNCH(ctx, k_center_ranks, 1, 1, 0, counts, rank, world, max_size, plan);
    URH_LAUNCH(ctx, k_center_window, nb, 256, 0, d_qad, n, ts, (const int64_t*)prefix, ntiles, plan, partial);
    const CenStats* parts = &plan->local;
    if (world > 1) {
        URH_TL_MARK(ctx, "x2 window partials: enter");
        URH_CHECK(urh_nccl_allgather(ctx, &plan->local, d_parts, sizeof(CenStats)));
        URH_TL_MARK(ctx, "x2 window partials: done");
        parts = d_parts;
    }
    URH_LAUNCH(ctx, k_center_plan, 1, 256, 0, parts, world, plan, fe, hist, xhist);
    const size_t dyn = (size_t)CEN_MAX_BINS * 4 + (size_t)(CEN_MAX_BINS + 3) * 4;   // histogram + edge table, 48 KB
    const unsigned gs = (unsigned)min(urh_div_up(ntiles, 8), (int64_t)ctx->sm_count * 8);
    // the window's cut tiles (and, with a fine histogram, the interior tiles of its cut slabs), then the certificate
    URH_LAUNCH(ctx, k_hist_window_ends, fine ? 2 + ctx->sm_count * 4 : 2, 256, fine ? dyn : 0, d_qad, n, (const int64_t*)prefix,
               (const CenterPlan*)plan, (const float*)fe, hist, xhist, fine ? fine->slab_tiles : (int64_t)1);
    if (fine) URH_LAUNCH(ctx, k_center_certify, 1, CERT_THREADS, 0, *fine, plan, (const float*)fe, (const unsigned long long*)xhist, cert_lo, cert_hi);
    URH_LAUNCH(ctx, (k_hist_interior<true, true, 3>), gs, 256, dyn, d_qad, n, (const CenterPlan*)plan, (const float*)fe, hist, (const int64_t*)prefix, 1);
    URH_LAUNCH(ctx, (k_hist_interior<true, false, 3>), gs, 256, dyn, d_qad, n, (const CenterPlan*)plan, (const float*)fe, hist, (const int64_t*)prefix, 1);
    if (world > 1) {
        URH_TL_MARK(ctx, "x3 histogram sum: enter");
        URH_CHECK(urh_nccl_allreduce_i64(ctx, (int64_t*)hist, CEN_MAX_BINS, 0));
        URH_TL_MARK(ctx, "x3 histogram sum: done");
    }
    URH_LAUNCH(ctx, k_center_pick, 1, 256, 0, (const unsigned long long*)hist, plan);
    ctx->center_prefix = prefix;
    ctx->center_ts = ts;
    ctx->center_n = n;
    ctx->center_x = d_qad;
    *d_plan_out = plan;
    return URH_OK;
}

// {certified, -, straddle mass} of a plan -> h_dst3 (pinned), on the stream
int urh_center_plan_certify_stats(urh_ctx* ctx, const CenterPlan* plan, int64_t* h_dst3) {
    h_dst3[0] = h_dst3[1] = h_dst3[2] = 0;
    URH_CUDA(ctx, cudaMemcpyAsync(h_dst3, &plan->certified, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_dst3 + 2, &plan->straddle, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    return URH_OK;
}

// certificate of the last one-call step: {1 if the fine histogram decided the center (no histogram pass over qad) else 0,
// buckets of the fine histogram (0: not collected), U - L summed over the two deciding bins}
extern "C" int urh_center_certify_stats(urh_ctx* ctx, int64_t* h_out3) {
    for (int i = 0; i < 3; i++) h_out3[i] = ctx->center_cert[i];
    return URH_OK;
}

// {center (double), state} of a plan -> 16 bytes at dst (device or pinned host), on the stream
int urh_center_plan_result(urh_ctx* ctx, const CenterPlan* plan, const float** d_centerf, const double** d_center, const int** d_state) {
    if (d_centerf) *d_centerf = &plan->centerf;
    if (d_center) *d_center = &plan->center;
    if (d_state) *d_state = &plan->state;
    return URH_OK;
}
