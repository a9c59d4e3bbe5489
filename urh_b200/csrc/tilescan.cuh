// Single-launch exclusive scan over a device table (decoupled look-back), for any associative — not necessarily
// commutative — operator; the library's one device-wide scan.  Most tables have one entry per TILE (the run-carry,
// candidate, firing and kept-count summaries of the dense pass's tiles); others have one per pulse row or per sample
// (ppseq_to_bits, detect_modulation's compaction).  The `load` and `post` hooks fold the element-wise kernels that
// would produce a scan's input or consume its output into the scan itself.  `post` may write the table `load` reads:
// a thread loads all its elements before it posts any, and no other thread touches them.
//
//   F::load(i)                  -> element i (computed on the fly from other tables)
//   F::post(i, excl, elem)      called for every i < n with its EXCLUSIVE prefix (identity for i == 0)
//   *d_total (optional)         the reduction of all elements (n <= 0: nothing is launched or written)
//
// Blocks take their chunk index from a monotonic counter in arrival order, so a block only ever waits for blocks
// that are already running (forward progress without co-residency assumptions).  The per-block status words carry
// a launch epoch: no memset between launches.
#pragma once
#include "common.cuh"

namespace urhts {

constexpr int BLOCK = 256;
constexpr int SLOT = 32;  // bytes reserved per published value (sizeof(T) <= SLOT, multiple of 4)

struct Ws {
    unsigned long long* counter;  // dynamic block ids (never reset)
    uint32_t* status;             // (epoch << 2) | {1: aggregate published, 2: inclusive prefix published}
    char* agg;
    char* pre;
    unsigned long long base;      // value of *counter when this launch's first block arrives
    uint32_t epoch;
};

template <typename T>
union Words {
    T v;
    uint32_t w[sizeof(T) / 4];
    __device__ __forceinline__ Words() {}
};

template <typename T>
__device__ __forceinline__ T shfl_up_t(const T& x, int d) {
    static_assert(sizeof(T) % 4 == 0 && sizeof(T) <= SLOT, "scan element: multiple of 4 bytes, at most SLOT");
    Words<T> a, r;
    a.v = x;
#pragma unroll
    for (int k = 0; k < (int)(sizeof(T) / 4); k++) r.w[k] = __shfl_up_sync(URH_FULL_MASK, a.w[k], d);
    return r.v;
}
template <typename T>
__device__ __forceinline__ T shfl_t(const T& x, int src) {
    Words<T> a, r;
    a.v = x;
#pragma unroll
    for (int k = 0; k < (int)(sizeof(T) / 4); k++) r.w[k] = __shfl_sync(URH_FULL_MASK, a.w[k], src);
    return r.v;
}
template <typename T>
__device__ __forceinline__ void publish(char* slots, int64_t b, const T& x) {
    Words<T> a;
    a.v = x;
    uint32_t* p = (uint32_t*)(slots + b * SLOT);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(T) / 4); k++) __stcg(p + k, a.w[k]);
}
template <typename T>
__device__ __forceinline__ T fetch(const char* slots, int64_t b) {
    Words<T> a;
    const uint32_t* p = (const uint32_t*)(slots + b * SLOT);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(T) / 4); k++) a.w[k] = __ldcg(p + k);
    return a.v;
}
__device__ __forceinline__ uint32_t ld_status(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_status(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ITEMS consecutive elements per thread.  The look-back chain advances 32 blocks per global-memory round trip, so few, fat
// blocks finish sooner than many thin ones on tables of this size (2^19 tiles: 128 blocks at ITEMS = 16).
template <typename T, typename Op, typename F, int ITEMS>
__global__ void __launch_bounds__(BLOCK) k_scan(int64_t n, T identity, Op op, F f, Ws ws, T* __restrict__ total_out) {
    constexpr int CHUNK = BLOCK * ITEMS;
    __shared__ unsigned long long s_bid;
    __shared__ T s_warp[BLOCK / 32];
    __shared__ T s_block_excl;
    if (threadIdx.x == 0) s_bid = atomicAdd(ws.counter, 1ull) - ws.base;
    __syncthreads();
    const int64_t bid = (int64_t)s_bid;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t first = bid * CHUNK + (int64_t)threadIdx.x * ITEMS;
    T v[ITEMS];
    T acc = identity;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        v[i] = (first + i < n) ? f.load(first + i) : identity;
        acc = op(acc, v[i]);
    }
    // inclusive scan of the thread aggregates inside the warp (order-preserving)
    T incl = acc;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const T o = shfl_up_t(incl, off);
        if (lane >= off) incl = op(o, incl);
    }
    T lane_excl = shfl_up_t(incl, 1);
    if (lane == 0) lane_excl = identity;
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        constexpr int NW = BLOCK / 32;
        T wi = (lane < NW) ? s_warp[lane] : identity;
#pragma unroll
        for (int off = 1; off < NW; off <<= 1) {
            const T o = shfl_up_t(wi, off);
            if (lane >= off) wi = op(o, wi);
        }
        T wex = shfl_up_t(wi, 1);
        if (lane == 0) wex = identity;
        const T block_agg = shfl_t(wi, NW - 1);
        T excl = identity;
        if (bid > 0) {
            if (lane == 0) {
                publish(ws.agg, bid, block_agg);
                __threadfence();
                st_status(ws.status + bid, (ws.epoch << 2) | 1u);
            }
            // look-back, 32 predecessors per round: lane j examines block look - j
            int64_t look = bid - 1;
            bool done = false;
            while (!done) {
                const int64_t p = look - lane;
                uint32_t st;
                bool ready;
                do {
                    st = (p >= 0) ? ld_status(ws.status + p) : ((ws.epoch << 2) | 2u);   // before block 0: the identity prefix
                    ready = (st >> 2) == ws.epoch && (st & 3u) != 0u;
                } while (!__all_sync(URH_FULL_MASK, ready));
                __threadfence();
                const bool is_pre = (st & 3u) == 2u;
                T val = identity;
                if (p >= 0) val = is_pre ? fetch<T>(ws.pre, p) : fetch<T>(ws.agg, p);
                const uint32_t pm = __ballot_sync(URH_FULL_MASK, is_pre);
                const int far = pm ? (__ffs(pm) - 1) : 31;   // farthest block folded this round
                T window = shfl_t(val, far);
                for (int j = far - 1; j >= 0; j--) window = op(window, shfl_t(val, j));
                excl = op(window, excl);
                done = pm != 0u;
                look -= 32;
            }
        }
        if (lane == 0) {
            const T inclusive = op(excl, block_agg);
            publish(ws.pre, bid, inclusive);
            __threadfence();
            st_status(ws.status + bid, (ws.epoch << 2) | 2u);
            s_block_excl = excl;
            if (total_out && (bid + 1) * (int64_t)CHUNK >= n) *total_out = inclusive;
        }
        if (lane < NW) s_warp[lane] = wex;
    }
    __syncthreads();
    T run = op(s_block_excl, op(s_warp[warp], lane_excl));
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        if (first + i < n) {
            f.post(first + i, run, v[i]);
            run = op(run, v[i]);
        }
    }
}

// host side (context.cu): workspace for `nblocks` blocks of the next launch.  The workspace starts at 8192 blocks (a table of
// 2^25 elements at ITEMS = 16, 2^24 at 8); a larger launch grows it once, which synchronises the context stream and reallocates.
int prepare(urh_ctx* ctx, int64_t nblocks, Ws* out);

struct AddI64 {
    __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a + b; }
};

template <typename T, typename Op, typename F, int ITEMS = 16>
static inline int scan(urh_ctx* ctx, int64_t n, T identity, Op op, F f, T* d_total) {
    if (n <= 0) return URH_OK;
    const int64_t nb = urh_div_up(n, (int64_t)BLOCK * ITEMS);
    Ws ws;
    URH_CHECK(prepare(ctx, nb, &ws));
    URH_LAUNCH(ctx, (k_scan<T, Op, F, ITEMS>), (unsigned)nb, BLOCK, 0, n, identity, op, f, ws, d_total);
    return URH_OK;
}

}  // namespace urhts
