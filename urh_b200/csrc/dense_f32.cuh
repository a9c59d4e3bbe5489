// Dense pass over an array of already-computed real samples (float32 / float64): classification + run
// tracking only.  Used by grab_pulse_lens (stand-alone), segment_messages_from_magnitudes and
// get_plateau_lengths.
#pragma once
#include "dense.cuh"

// Classifier sources for the stand-alone digitizer / segmenter: float32 samples already in memory.
// BINARY sources also give the class as two predicates (noise, above) for UrhRunTracker::feed_masks.
struct SrcQad {  // grab_pulse_lens on a demodulated array
    static constexpr bool BINARY = false;
    template <typename T> __device__ __forceinline__ static int cls(T s, const UrhClassify& C, float) { return urh_classify((float)s, C); }
    template <typename T> __device__ __forceinline__ static void bits(T, const UrhClassify&, float, bool& nz, bool& ab) { nz = false; ab = false; }
    template <typename T> __device__ __forceinline__ static bool above(T, float) { return false; }
};
struct SrcQad2 {  // the same for a binary digitizer (order 2): no threshold loop, no branches
    static constexpr bool BINARY = true;
    template <typename T> __device__ __forceinline__ static int cls(T s, const UrhClassify& C, float thr0) {
        const int c = ((float)s <= thr0) ? 0 : 1;
        return ((float)s == C.noise_value) ? -1 : c;
    }
    template <typename T> __device__ __forceinline__ static void bits(T s, const UrhClassify& C, float thr0, bool& nz, bool& ab) {
        nz = (float)s == C.noise_value;
        ab = !((float)s <= thr0) && !nz;
    }
    template <typename T> __device__ __forceinline__ static bool above(T s, float thr0) { return !((float)s <= thr0); }   // tile without noise
};
struct SrcAbove {  // segment_messages_from_magnitudes: class 1 = above noise (auto_interpretation.pyx:79)
    static constexpr bool BINARY = true;
    template <typename T> __device__ __forceinline__ static int cls(T s, const UrhClassify&, float thr0) { return (s > (T)thr0) ? 1 : 0; }
    template <typename T> __device__ __forceinline__ static void bits(T s, const UrhClassify&, float thr0, bool& nz, bool& ab) { nz = false; ab = s > (T)thr0; }
    template <typename T> __device__ __forceinline__ static bool above(T s, float thr0) { return s > (T)thr0; }
};
struct SrcCenter {  // get_plateau_lengths: -1/1 around center (auto_interpretation.pyx:183,197) as 0/1
    static constexpr bool BINARY = true;
    template <typename T> __device__ __forceinline__ static int cls(T s, const UrhClassify&, float thr0) { return (s <= (T)thr0) ? 0 : 1; }
    template <typename T> __device__ __forceinline__ static void bits(T s, const UrhClassify&, float thr0, bool& nz, bool& ab) { nz = false; ab = !(s <= (T)thr0); }
    template <typename T> __device__ __forceinline__ static bool above(T s, float thr0) { return !(s <= (T)thr0); }
};

// Speculative digitizing of the detect-center step (DESIGN.md §4.4.1): the demodulation pass digitized tiles [lo, hi) at the
// guess *tg and left margin[t] = min over tile t of fl(|s - t_g|).  At the real threshold c a kept sample changes class only if it
// lies in (t_g, c] or (c, t_g]; rounding is monotone, so then fl(|s - t_g|) <= fl(|c - t_g|).  margin[t] > fl(|c - t_g|) therefore
// proves every class of tile t unchanged, and the summary and staging the pass wrote are exactly the ones this kernel would write.
struct UrhSpec {
    const float* tg;
    float* margin;
    int64_t lo, hi;          // lo == hi: nothing speculated
    unsigned int* redone;    // speculated tiles that failed the proof and were digitized again
};

template <typename T> struct UrhVec2;
template <> struct UrhVec2<float> { typedef float2 type; };
template <> struct UrhVec2<double> { typedef double2 type; };

// One tile (warp-uniform): classify, track runs, write the summary and the staged candidates.
template <typename SRC, typename T>
__device__ __forceinline__ void dense_f32_tile(const T* __restrict__ x, int64_t n, int vec_in, const UrhClassify& cls, float thr0, int tol,
                                               UrhTileSummary* __restrict__ tiles, uint32_t* __restrict__ staging, int stage_cap,
                                               int16_t* __restrict__ init_cls, int cls_of_zero, const UrhTileStats* __restrict__ tile_stats,
                                               int64_t tile, int lane) {
    const int64_t tile_start = tile * URH_TILE;
    const int tile_len = (int)((n - tile_start) < URH_TILE ? (n - tile_start) : URH_TILE);
    const int iters = (tile_len + 63) >> 6;
    UrhRunTracker rt;
    rt.init(tol, staging + tile * (int64_t)stage_cap);
    if (vec_in && tile_len == URH_TILE) {
        // full tile: eight 64-groups in flight per warp (four being classified, four being loaded)
        typedef typename UrhVec2<T>::type V;
        const V* p = (const V*)(x + tile_start) + lane;  // 64-group `it` -> p[it * 32]
        constexpr int ITERS = URH_TILE / 64;
        // the demodulator counted the tile's kept samples (> -4): all kept <=> no sample carries the noise sentinel (<= -4), and
        // the noise masks (half of the compares, votes and mask arithmetic) are known to be zero
        const bool no_noise = SRC::BINARY && tile_stats && cls.noise_value <= -4.0f && tile_stats[tile].cnt == URH_TILE;
        // eight 64-groups in flight per warp (four being classified, four being loaded)
        V cur[4], nxt[4];
#pragma unroll
        for (int j = 0; j < 4; j++) cur[j] = __ldg(p + j * 32);
        if (tile_start == 0 && lane == 0 && init_cls) *init_cls = (int16_t)(((float)cur[0].x == cls.noise_value) ? -1 : cls_of_zero);
        if (SRC::BINARY) {
            // stream the tile into class masks (lane g keeps group g's), settle the whole tile afterwards
            UrhTileResolve tr;
            tr.init();
#pragma unroll 1
            for (int it = 0; it < ITERS; it += 4) {
                if (it + 4 < ITERS) {
#pragma unroll
                    for (int j = 0; j < 4; j++) nxt[j] = __ldg(p + (it + 4 + j) * 32);
                }
                if (no_noise) {
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        tr.keep(it + j, 0u, __ballot_sync(URH_FULL_MASK, SRC::template above<T>(cur[j].x, thr0)), 0u,
                                __ballot_sync(URH_FULL_MASK, SRC::template above<T>(cur[j].y, thr0)), lane);
                } else {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        bool nx, ax, ny, ay;
                        SRC::template bits<T>(cur[j].x, cls, thr0, nx, ax);
                        SRC::template bits<T>(cur[j].y, cls, thr0, ny, ay);
                        tr.keep(it + j, __ballot_sync(URH_FULL_MASK, nx), __ballot_sync(URH_FULL_MASK, ax), __ballot_sync(URH_FULL_MASK, ny),
                                __ballot_sync(URH_FULL_MASK, ay), lane);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; j++) cur[j] = nxt[j];
            }
            tr.finish(tol, staging + tile * (int64_t)stage_cap, tiles + tile, lane);
            return;
        }
#pragma unroll 1
        for (int it = 0; it < ITERS; it += 4) {
            if (it + 4 < ITERS) {
#pragma unroll
                for (int j = 0; j < 4; j++) nxt[j] = __ldg(p + (it + 4 + j) * 32);
            }
#pragma unroll
            for (int j = 0; j < 4; j++)
                rt.feed(it + j, SRC::template cls<T>(cur[j].x, cls, thr0), SRC::template cls<T>(cur[j].y, cls, thr0), true, true, lane);
#pragma unroll
            for (int j = 0; j < 4; j++) cur[j] = nxt[j];
        }
        rt.finish(tile_len, tiles + tile, lane);
        return;
    }
    // two 64-groups in flight per warp step
    for (int it = 0; it < iters; it += 2) {
        T a0 = 0, a1 = 0, b0 = 0, b1 = 0;
        const int64_t pa = tile_start + (int64_t)it * 64 + 2 * lane;
        const int64_t pb = pa + 64;
        if (vec_in && pa + 1 < n) {
            const typename UrhVec2<T>::type v = __ldg((const typename UrhVec2<T>::type*)(x + pa));
            a0 = v.x; a1 = v.y;
        } else {
            if (pa < n) a0 = __ldg(x + pa);
            if (pa + 1 < n) a1 = __ldg(x + pa + 1);
        }
        const bool has_b = it + 1 < iters;
        if (has_b) {
            if (vec_in && pb + 1 < n) {
                const typename UrhVec2<T>::type v = __ldg((const typename UrhVec2<T>::type*)(x + pb));
                b0 = v.x; b1 = v.y;
            } else {
                if (pb < n) b0 = __ldg(x + pb);
                if (pb + 1 < n) b1 = __ldg(x + pb + 1);
            }
        }
        if (pa == 0 && init_cls) *init_cls = (int16_t)(((float)a0 == cls.noise_value) ? -1 : cls_of_zero);
        rt.feed(it, SRC::template cls<T>(a0, cls, thr0), SRC::template cls<T>(a1, cls, thr0), pa < n, pa + 1 < n, lane);
        if (has_b) rt.feed(it + 1, SRC::template cls<T>(b0, cls, thr0), SRC::template cls<T>(b1, cls, thr0), pb < n, pb + 1 < n, lane);
    }
    rt.finish(tile_len, tiles + tile, lane);
}

// Warp-stride loop over tiles: warp w digitizes tiles w, w + W, w + 2W, ... (W warps in the grid).  A grid of one warp per tile runs
// the loop once per warp; the detect step's pass after speculation runs a grid sized to the GPU, because it redoes a handful of tiles
// and one block per eight tiles would cost more in block launches than the work.  Lane i triages the warp's (i+1)-th next tile, so
// the checks that skip a tile cost one load per 32 tiles: an all-NOISE tile first, then the speculation proof, then the count.
template <typename SRC, typename T>
__global__ void __launch_bounds__(URH_WARPS_PER_BLOCK * 32)
k_dense_f32(const T* __restrict__ x, int64_t n, int vec_in, const __grid_constant__ UrhClassify cls, int tol,
            UrhTileSummary* __restrict__ tiles, uint32_t* __restrict__ staging, int stage_cap,
            int16_t* __restrict__ init_cls, int cls_of_zero, const float* __restrict__ d_thr0 = nullptr,
            const UrhTileStats* __restrict__ tile_stats = nullptr, const UrhSpec spec = UrhSpec{}) {
    // d_thr0: the (binary) threshold lives in device memory (center detected on the device); then cls_of_zero is derived here
    const float thr0 = d_thr0 ? *d_thr0 : cls.thr[0];
    if (d_thr0) cls_of_zero = (0.0f <= thr0) ? 0 : 1;
    const int lane = threadIdx.x & 31;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    const int64_t stride = (int64_t)gridDim.x * URH_WARPS_PER_BLOCK;
    for (int64_t t0 = (int64_t)blockIdx.x * URH_WARPS_PER_BLOCK + (threadIdx.x >> 5); t0 < ntiles; t0 += 32 * stride) {
        const int64_t mine = t0 + lane * stride;
        bool work = mine < ntiles;
        if (work && tile_stats && tile_stats[mine].all_noise) {
            // the demodulator's tile table says the whole tile is NOISE: one run of class -1, nothing to read (captures are mostly silence)
            const int64_t rem = n - mine * URH_TILE;
            const int tile_len = rem < URH_TILE ? (int)rem : URH_TILE;
            UrhTileSummary s;
            s.first_cls = -1; s.last_cls = -1; s.head_len = tile_len; s.tail_len = tile_len; s.ncand = 0;
            tiles[mine] = s;
            if (mine == 0 && init_cls) *init_cls = (int16_t)-1;
            work = false;
        } else if (work && mine >= spec.lo && mine < spec.hi) {
            // the demodulation pass digitized the tile at the guess t_g: keep its result when the margin proves the classes (UrhSpec)
            if (spec.margin[mine] > fabsf(__fsub_rn(thr0, *spec.tg))) work = false;
            else atomicAdd(spec.redone, 1u);
        }
        for (unsigned m = __ballot_sync(URH_FULL_MASK, work); m; m &= m - 1)
            dense_f32_tile<SRC, T>(x, n, vec_in, cls, thr0, tol, tiles, staging, stage_cap, init_cls, cls_of_zero, tile_stats,
                                   t0 + (int64_t)(__ffs(m) - 1) * stride, lane);
    }
}
