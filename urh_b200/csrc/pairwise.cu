// numpy's float32 pairwise summation, replayed in parallel — so that detect_center's `np.var(rect)`
// (AutoInterpretation.py:240: the histogram's bin width) comes out BIT-IDENTICAL on the GPU.
//
// What numpy computes (numpy/_core/src/umath/loops_utils.h.src @TYPE@_pairwise_sum, _methods.py _var; restated and pinned
// bit-for-bit against numpy by tests/test_pairwise_model.py):
//   sum(a, n):  n < 8    : r = 0; r += a[i] in order
//               n <= 128 : eight accumulators r[k] = a[k]; r[k] += a[i + k] for i = 8, 16, ... while i < n - n % 8;
//                          res = ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)); then res += a[i] for the remaining n % 8
//               else     : n2 = n/2 - (n/2) % 8;  sum(a, n2) + sum(a + n2, n - n2)
//   add.reduce = 0.0f + sum(a, n)
//   mean = float32(double(add.reduce(a)) / n);  x = (a - mean)^2 in float32;  var = float32(double(add.reduce(x)) / n)
// The split points depend on n only, so the tree is known up front: a leaf is 64 < len <= 128 consecutive elements and the
// leaves sit at most D levels deep (D ~ log2(n / 64)).  One 8-lane group per leaf reproduces the eight accumulators (lane k =
// accumulator k, combined by xor-shuffles 1, 2, 4 = numpy's bracket), then the tree is folded level by level.
//
// Layout: "slot" j in [0, 2^D) = the path from the root (bit D-1-d of j = right turn at depth d).  A leaf at depth d <= D
// covers 2^(D-d) slots and stores its sum at its first slot; depth_of[j] = depth of the leaf covering slot j.
#include "dense.cuh"

struct PwNode {
    int64_t start, len;
    int depth;
};

// descend from the root (0, n) along the bits of slot j until a leaf (len <= 128) is reached
__device__ __forceinline__ PwNode pw_descend(int64_t n, int D, int64_t j) {
    PwNode nd;
    nd.start = 0; nd.len = n; nd.depth = 0;
    while (nd.len > 128) {
        int64_t n2 = nd.len / 2;
        n2 -= n2 % 8;
        const int right = (int)((j >> (D - 1 - nd.depth)) & 1);
        if (right) { nd.start += n2; nd.len -= n2; }
        else nd.len = n2;
        nd.depth++;
    }
    return nd;
}

// element i of the summed sequence: the window sample itself (MODE 0) or its float32 squared deviation from `mean` (MODE 1)
template <int MODE>
__device__ __forceinline__ float pw_elem(const float* __restrict__ a, int64_t i, float mean) {
    const float v = a[i];
    if (MODE == 0) return v;
    const float d = __fsub_rn(v, mean);
    return __fmul_rn(d, d);
}

// one 8-lane group per slot; only the group of a leaf's FIRST slot does the work.  Batch b = blockIdx.y sums the n elements
// from a + off0 + b * step into val[b << D ...]; every batch has the same tree, so batch 0 alone writes depth_of.
template <int MODE>
__global__ void __launch_bounds__(256) k_pw_leaves(const float* __restrict__ a, int64_t n, int D, const float* __restrict__ d_mean,
                                                  float* __restrict__ val, uint8_t* __restrict__ depth_of, int64_t off0, int64_t step) {
    const int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;   // slot
    const int k = threadIdx.x & 7;
    const unsigned gmask = 0xffu << ((threadIdx.x & 31) & ~7);
    if (g >= ((int64_t)1 << D)) return;
    const float mean = MODE ? *d_mean : 0.0f;
    const PwNode nd = pw_descend(n, D, g);
    if (k == 0 && blockIdx.y == 0) depth_of[g] = (uint8_t)nd.depth;
    const int64_t first = (nd.depth < D) ? ((g >> (D - nd.depth)) << (D - nd.depth)) : g;
    if (g != first) return;
    const float* p = a + off0 + (int64_t)blockIdx.y * step;
    val += (int64_t)blockIdx.y << D;
    const int64_t s = nd.start;
    const int len = (int)nd.len;
    float res;
    if (len < 8) {
        res = 0.0f;
        if (k == 0)
            for (int i = 0; i < len; i++) res = __fadd_rn(res, pw_elem<MODE>(p, s + i, mean));
    } else {
        float r = pw_elem<MODE>(p, s + k, mean);
        const int body = len - (len % 8);
        for (int i = 8; i < body; i += 8) r = __fadd_rn(r, pw_elem<MODE>(p, s + i + k, mean));
        r = __fadd_rn(r, __shfl_xor_sync(gmask, r, 1));
        r = __fadd_rn(r, __shfl_xor_sync(gmask, r, 2));
        r = __fadd_rn(r, __shfl_xor_sync(gmask, r, 4));
        res = r;
        if (k == 0)
            for (int i = body; i < len; i++) res = __fadd_rn(res, pw_elem<MODE>(p, s + i, mean));
    }
    if (k == 0) val[g] = res;
}

// fold level d (nodes at depth d, 2^d of them): node j is internal iff the leaf covering its first slot lies deeper than d
__global__ void k_pw_level(float* __restrict__ val, const uint8_t* __restrict__ depth_of, int D, int d) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ((int64_t)1 << d)) return;
    val += (int64_t)blockIdx.y << D;   // batch
    const int64_t left = j << (D - d);
    if (depth_of[left] <= d) return;
    const int64_t right = left + ((int64_t)1 << (D - d - 1));
    val[left] = __fadd_rn(val[left], val[right]);
}

// the top levels (d < top) in one block per batch; then out[2b] = 0.0f + sum, out[2b + 1] = float32(double(that) / n)
__global__ void __launch_bounds__(1024) k_pw_top(float* __restrict__ val, const uint8_t* __restrict__ depth_of, int D, int top, int64_t n,
                                                float* __restrict__ out) {
    val += (int64_t)blockIdx.x << D;
    for (int d = top - 1; d >= 0; d--) {
        for (int64_t j = threadIdx.x; j < ((int64_t)1 << d); j += blockDim.x) {
            const int64_t left = j << (D - d);
            if (depth_of[left] > d) {
                const int64_t right = left + ((int64_t)1 << (D - d - 1));
                val[left] = __fadd_rn(val[left], val[right]);
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float s = __fadd_rn(0.0f, val[0]);   // add.reduce starts from the identity
        out[2 * blockIdx.x] = s;
        out[2 * blockIdx.x + 1] = __double2float_rn(__ddiv_rn((double)s, (double)n));
    }
}

static int pw_depth(int64_t n) {
    // depth of the deepest leaf: follow the larger (right) child
    int d = 0;
    while (n > 128) {
        int64_t n2 = n / 2;
        n2 -= n2 % 8;
        n -= n2;
        d++;
    }
    return d;
}

// d_out[2b] = add.reduce of the n elements from d_a + off0 + b * step, d_out[2b + 1] = float32(double(sum) / n), b < batch.
// MODE 1 reads the mean from d_mean (device).
template <int MODE>
static int pw_reduce(urh_ctx* ctx, const float* d_a, int64_t n, const float* d_mean, float* d_out, int batch = 1, int64_t off0 = 0,
                     int64_t step = 0) {
    const int D = pw_depth(n);
    const int64_t slots = (int64_t)1 << D;
    float* val;
    uint8_t* depth_of;
    URH_CHECK(urh_arena(ctx, (size_t)slots * batch, &val));
    URH_CHECK(urh_arena(ctx, (size_t)slots, &depth_of));
    URH_LAUNCH(ctx, (k_pw_leaves<MODE>), dim3((unsigned)urh_div_up(slots * 8, 256), (unsigned)batch), 256, 0, d_a, n, D, d_mean, val,
               depth_of, off0, step);
    const int top = D < 12 ? D : 12;
    for (int d = D - 1; d >= top; d--)
        URH_LAUNCH(ctx, k_pw_level, dim3((unsigned)urh_div_up((int64_t)1 << d, 256), (unsigned)batch), 256, 0, val,
                   (const uint8_t*)depth_of, D, d);
    URH_LAUNCH(ctx, k_pw_top, (unsigned)batch, 1024, 0, val, (const uint8_t*)depth_of, D, top, n, d_out);
    return URH_OK;
}

// np.mean's float32 sums of the `batch` equal-length chunks [n - (b+1)*len, n - b*len) of d_a (detect_noise_level's end-aligned
// 1 % chunks of a float32 magnitude array): d_out[2b] = numpy's pairwise sum of chunk b, d_out[2b + 1] = float32(sum / len).
int urh_chunk_sums_f32(urh_ctx* ctx, const float* d_a, int64_t n, int64_t len, int batch, float* d_out) {
    return pw_reduce<0>(ctx, d_a, len, nullptr, d_out, batch, n - len, -len);
}

// ---- compaction of the rank window ------------------------------------------------------------------------------------------
// out[rank - r0] = the kept samples (x > -4) of local rank r0 <= rank < r1, in order.  One warp per tile of [t0, t1].
__global__ void __launch_bounds__(256) k_compact_window(const float* __restrict__ x, int64_t n, const int64_t* __restrict__ prefix,
                                                       int64_t t0, int64_t t1, int64_t r0, int64_t r1, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t t = t0 + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (t > t1) return;
    int64_t rank = prefix[t];
    if (prefix[t + 1] == rank || prefix[t + 1] <= r0 || rank >= r1) return;   // no kept sample / entirely outside the window
    const int64_t base = t * URH_TILE;
    for (int it = 0; it < URH_TILE / 32; it++) {
        const int64_t i = base + it * 32 + lane;
        const float v = (i < n) ? x[i] : -5.0f;
        const bool kept = v > -4.0f;
        const unsigned m = __ballot_sync(URH_FULL_MASK, kept);
        const int64_t mine = rank + __popc(m & ((1u << lane) - 1u));
        if (kept && mine >= r0 && mine < r1) out[mine - r0] = v;
        rank += __popc(m);
    }
}

// np.var of the rank window [r0, r1) of the kept samples of d_x, exactly as numpy computes it for a float32 array.
// prefix = kept-sample rank prefix of the tiles (ntiles + 1 entries, arena); win tiles [t0, t1] hold the window.
// h_out2 = {mean, var} (float32 values).
int urh_window_var_bitwise(urh_ctx* ctx, const float* d_x, int64_t n, const int64_t* d_prefix, int64_t t0, int64_t t1, int64_t r0,
                           int64_t r1, float* h_out2) {
    const int64_t W = r1 - r0;
    h_out2[0] = h_out2[1] = 0.0f;
    if (W <= 0) return URH_OK;
    float* rect;
    float* d_res;
    URH_CHECK(urh_arena(ctx, (size_t)W, &rect));
    URH_CHECK(urh_arena(ctx, 4, &d_res));
    URH_LAUNCH(ctx, k_compact_window, (unsigned)urh_div_up(t1 - t0 + 1, 8), 256, 0, d_x, n, d_prefix, t0, t1, r0, r1, rect);
    URH_CHECK((pw_reduce<0>(ctx, rect, W, nullptr, d_res)));           // d_res[1] = mean
    URH_CHECK((pw_reduce<1>(ctx, rect, W, d_res + 1, d_res + 2)));     // d_res[3] = var
    float h[4];
    URH_CUDA(ctx, cudaMemcpyAsync(h, d_res, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h_out2[0] = h[1];
    h_out2[1] = h[3];
    return URH_OK;
}
