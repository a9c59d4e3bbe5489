// FIR filtering and DC correction (reference: signal_functions.fir_filter signal_functions.pyx:513-525,
// Filter.work / apply_fir_filter / apply_bandpass_filter Filter.py:31-46, 84-101).
//
// fir_filter is reproduced in the reference's exact accumulation order: y[k] = sum over i ascending of
// x[i]*taps[k-i], every complex64 product and every add individually rounded (no FMA) — bit-identical output, non-finite
// samples and taps included (see urh_fir_filter).
// A block stages its input tile (outputs + M-1 halo samples) in shared memory with cp.async.bulk (TMA 1-D bulk
// copy, mbarrier completion); each thread then produces 4 consecutive outputs so that every tap fetched from
// shared memory is used four times.  This kernel is FP32-ALU-bound (8*M unfused flops per sample), not
// HBM-bound: SURVEY §8d reports FP32 utilisation for it.
//
// The band-pass path (complex128 taps, numpy 'same'/FFT convolution in the reference) is evaluated as a
// direct convolution with double accumulation — the reference's own result is a complex128 FFT product, so
// parity is tolerance-based (1e-5 of the signal scale) as stated in BASELINE.md.
#include "common.cuh"
#include "stream_ring.cuh"

#include <cuda/barrier>
#include <math.h>

#define FIR_THREADS 256
#define FIR_PER_THREAD 4
#define FIR_TILE (FIR_THREADS * FIR_PER_THREAD)

__device__ __forceinline__ void fir_mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void fir_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes));
}
__device__ __forceinline__ void fir_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (uint32_t)__cvta_generic_to_shared(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
                 : "memory");
}
__device__ __forceinline__ void fir_mbar_wait(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"((uint32_t)__cvta_generic_to_shared(bar)),
        "r"(phase));
}

// One output as the reference computes it: +0, then x[k - q] * taps[q] for q = qmax .. 0 (ascending input index), each product
// std::complex<float>'s (urh_cmulf, with the Annex G recovery) and each add rounded.  xk points at x[k]; qmax leaves out the zero
// initial state.  The kernels below call it only for an output whose fast sum has both parts NaN (see urh_fir_filter).
__device__ __noinline__ float2 fir_exact_output(const float2* xk, const float2* taps, int qmax) {
    float2 acc = make_float2(0.f, 0.f);
    for (int q = qmax; q >= 0; q--) {
        const float2 v = xk[-q], h = taps[q];
        float pr, pi;
        urh_cmulf(v.x, v.y, h.x, h.y, pr, pi);
        acc.x = __fadd_rn(acc.x, pr);
        acc.y = __fadd_rn(acc.y, pi);
    }
    return acc;
}

// Exact-order complex64 FIR.  smem: [taps M float2][tile FIR_TILE + M - 1 float2]
// HISTORY: x[-(m-1) .. -1] hold real samples (the previous shard's tail) and are read instead of the zero initial state.
template <bool HISTORY>
__global__ void __launch_bounds__(FIR_THREADS) k_fir_exact(const float2* __restrict__ x, int64_t n, const float2* __restrict__ taps,
                                                            int m, float2* __restrict__ y) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar;
    float2* s_taps = (float2*)smem_raw;
    float2* s_x = s_taps + ((m + 1) & ~1);  // keep 16-byte alignment of the tile
    const int64_t tile0 = (int64_t)blockIdx.x * FIR_TILE;
    const int64_t first = tile0 - (m - 1);          // first input sample the tile needs (may be < 0)
    const int64_t lo = (HISTORY || first >= 0) ? first : 0;
    const int64_t hi = min(tile0 + FIR_TILE, n);    // one past the last input sample
    const int halo_missing = (int)(lo - first);     // zero initial state: samples before the capture are 0 (none with HISTORY)
    for (int j = threadIdx.x; j < m; j += FIR_THREADS) s_taps[j] = taps[j];
    for (int j = threadIdx.x; j < halo_missing; j += FIR_THREADS) s_x[j] = make_float2(0.f, 0.f);
    // bulk-copy [lo, hi) into s_x + halo_missing: needs 16-byte aligned addresses and size
    const int64_t cnt = hi - lo;
    const bool bulk_ok = (((uintptr_t)(x + lo)) % 16 == 0) && ((halo_missing % 2) == 0) && (cnt % 2 == 0) && cnt > 0;
    if (threadIdx.x == 0) {
        fir_mbar_init(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (bulk_ok) {
        if (threadIdx.x == 0) {
            fir_mbar_expect_tx(&bar, (uint32_t)(cnt * sizeof(float2)));
            fir_bulk_g2s(s_x + halo_missing, x + lo, (uint32_t)(cnt * sizeof(float2)), &bar);
        }
        fir_mbar_wait(&bar, 0);
    } else {
        for (int64_t j = threadIdx.x; j < cnt; j += FIR_THREADS) s_x[halo_missing + j] = x[lo + j];
    }
    __syncthreads();
    // thread t -> outputs k = tile0 + 4t .. 4t+3 ; s_x[j] holds x[first + j], so x[k - q] = s_x[k - q - first]
    const int64_t k0 = tile0 + (int64_t)threadIdx.x * FIR_PER_THREAD;
    if (k0 >= n) return;
    float2 acc[FIR_PER_THREAD];
#pragma unroll
    for (int r = 0; r < FIR_PER_THREAD; r++) acc[r] = make_float2(0.f, 0.f);
    // ascending input index i  <=>  descending tap index q = k - i, from q = m-1 down to 0
    const int base = (int)(k0 - first);  // s_x index of x[k0]
    for (int q = m - 1; q >= 0; q--) {
        const float2 h = s_taps[q];
#pragma unroll
        for (int r = 0; r < FIR_PER_THREAD; r++) {
            const float2 v = s_x[base + r - q];
            // complex64 product then += , each operation rounded (GCC's std::complex<float> without fast-math)
            const float pr = __fsub_rn(__fmul_rn(v.x, h.x), __fmul_rn(v.y, h.y));
            const float pi = __fadd_rn(__fmul_rn(v.x, h.y), __fmul_rn(v.y, h.x));
            acc[r].x = __fadd_rn(acc[r].x, pr);
            acc[r].y = __fadd_rn(acc[r].y, pi);
        }
    }
#pragma unroll
    for (int r = 0; r < FIR_PER_THREAD; r++)
        if (k0 + r < n) y[k0 + r] = acc[r];
    // both parts NaN: a product may have needed the Annex G recovery or been a padded 0 * non-finite tap (urh_fir_filter).  Such
    // outputs are redone from global memory after the stores, so that nothing but a 4-bit mask lives past the tap loop.
    unsigned redo = 0;
#pragma unroll
    for (int r = 0; r < FIR_PER_THREAD; r++)
        if (k0 + r < n && isnan(acc[r].x) && isnan(acc[r].y)) redo |= 1u << r;
    for (int r = 0; redo; r++, redo >>= 1)
        if (redo & 1) y[k0 + r] = fir_exact_output(x + k0 + r, taps, HISTORY ? m - 1 : (int)min((int64_t)m - 1, k0 + r));
}

// The same sums for tap counts whose tile does not fit in shared memory: one output per thread, taps and samples read from global
// memory, the real terms only (no zero initial state), the same descending q and the same recheck.
template <bool HISTORY>
__global__ void __launch_bounds__(FIR_THREADS) k_fir_exact_global(const float2* __restrict__ x, int64_t n, const float2* __restrict__ taps,
                                                                   int m, float2* __restrict__ y) {
    const int64_t k = (int64_t)blockIdx.x * FIR_THREADS + threadIdx.x;
    if (k >= n) return;
    const int qmax = HISTORY ? m - 1 : (int)min((int64_t)m - 1, k);
    float2 acc = make_float2(0.f, 0.f);
    for (int q = qmax; q >= 0; q--) {
        const float2 v = x[k - q], h = taps[q];
        const float pr = __fsub_rn(__fmul_rn(v.x, h.x), __fmul_rn(v.y, h.y));
        const float pi = __fadd_rn(__fmul_rn(v.x, h.y), __fmul_rn(v.y, h.x));
        acc.x = __fadd_rn(acc.x, pr);
        acc.y = __fadd_rn(acc.y, pi);
    }
    if (isnan(acc.x) && isnan(acc.y)) acc = fir_exact_output(x + k, taps, qmax);
    y[k] = acc;
}

#define FIR_SMEM_MAX (200 * 1024)

template <bool HISTORY>
static int fir_launch(urh_ctx* ctx, const float* d_x, int64_t n, const float* d_taps, int m, float* d_y) {
    const size_t smem = (size_t)(((m + 1) & ~1) + FIR_TILE + m - 1 + 2) * sizeof(float2);
    if (smem > FIR_SMEM_MAX) {   // m >= 12288
        URH_LAUNCH(ctx, k_fir_exact_global<HISTORY>, (unsigned)urh_div_up(n, FIR_THREADS), FIR_THREADS, 0, (const float2*)d_x, n,
                   (const float2*)d_taps, m, (float2*)d_y);
        return URH_OK;
    }
    URH_CUDA(ctx, cudaFuncSetAttribute(k_fir_exact<HISTORY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    URH_LAUNCH(ctx, k_fir_exact<HISTORY>, (unsigned)urh_div_up(n, FIR_TILE), FIR_THREADS, smem, (const float2*)d_x, n, (const float2*)d_taps, m,
               (float2*)d_y);
    return URH_OK;
}

// replaces signal_functions.fir_filter: x, y complex64[n] (device), taps complex64[m] (device)
extern "C" int urh_fir_filter(urh_ctx* ctx, const float* d_x, int64_t n, const float* d_taps, int m, float* d_y) {
    if (n <= 0) return URH_OK;
    if (m <= 0) {
        URH_CUDA(ctx, cudaMemsetAsync(d_y, 0, (size_t)n * 8, ctx->stream));
        return URH_OK;
    }
    // Why k_fir_exact's fast loop plus its recheck gives the reference's words.  The reference adds x[i] * taps[k - i] for its real
    // samples only, to an output that starts at +0 (np.zeros), each product a std::complex<float> product (__mulsc3).  The fast loop
    // multiplies naively and, for the first m-1 outputs, first adds the products of the zero initial state x[-1], x[-2], ...
    // * A naive product differs from __mulsc3's only when both of its parts are NaN (only then does the recovery run).
    // * A padded product 0 * taps[q] is +-0 in both parts when taps[q] is finite: added to +0 it leaves +0, so the real terms then
    //   meet the accumulator the reference starts from.  When taps[q] is infinite or NaN, it is NaN in both parts.
    // * Either exception makes both parts of the sum NaN, and NaN absorbs every later add.  So a sum that is not NaN in both parts
    //   saw neither: it is the reference's sum.  A sum that is NaN in both parts is recomputed over its real terms with urh_cmulf
    //   (fir_exact_output), in the same order.  Such outputs need a non-finite sample, tap or overflow, so the fast loop is untouched.
    // HISTORY (a shard after the first) has no padding, so only the recovery applies.  Beyond the shared-memory tile
    // (m >= 12288) k_fir_exact_global computes the same sums from global memory.
    return fir_launch<false>(ctx, d_x, n, d_taps, m, d_y);
}

// One shard of a capture cut by contiguous sample range: has_history != 0 means d_x[-(m-1) .. -1] hold the previous shard's last
// m-1 samples, so y equals urh_fir_filter of the whole capture from this shard's first sample on (same products, same order).
// has_history == 0 is urh_fir_filter itself (the first shard: zero initial state).
extern "C" int urh_fir_filter_shard(urh_ctx* ctx, const float* d_x, int64_t n, int has_history, const float* d_taps, int m, float* d_y) {
    if (!has_history || m <= 1) return urh_fir_filter(ctx, d_x, n, d_taps, m, d_y);
    if (n <= 0) return URH_OK;
    return fir_launch<true>(ctx, d_x, n, d_taps, m, d_y);
}

// Direct convolution sample c[t + offset], c = full convolution of x (complex64) with h (complex128 taps),
// double accumulation, complex64 result (band-pass path).
__global__ void k_conv_c128(const float2* __restrict__ x, int64_t n, const double2* __restrict__ h, int m, int64_t offset,
                            int64_t out_len, float2* __restrict__ y) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < out_len; k += stride) {
        const int64_t t = k + offset;
        double re = 0.0, im = 0.0;
        const int jlo = (int)max((int64_t)0, t - (n - 1)), jhi = (int)min((int64_t)m - 1, t);
        for (int j = jlo; j <= jhi; j++) {
            const float2 v = x[t - j];
            const double2 c = h[j];
            re += (double)v.x * c.x - (double)v.y * c.y;
            im += (double)v.x * c.y + (double)v.y * c.x;
        }
        y[k] = make_float2((float)re, (float)im);
    }
}

// The same convolution, tiled: the block converts its input span to double ONCE into shared memory (the naive kernel
// converts every sample once per tap -- the float->double converter, not the FMA pipe, was its limit), the taps sit in
// shared memory too, and every thread produces CONV_PER consecutive outputs from a sliding register window: one 16-byte
// shared-memory read feeds 4 * CONV_PER double FMAs.  CONV_PER is odd so that the lanes' 16-byte reads (stride CONV_PER * 16 B)
// fall into distinct banks.  Same accumulation order per output as k_conv_c128 (ascending tap index, fused multiply-adds).
#define CONV_PER 5
#define CONV_THREADS 256
#define CONV_TILE (CONV_PER * CONV_THREADS)
#define CONV_MAX_TAPS 768
__global__ void __launch_bounds__(CONV_THREADS) k_conv_c128_tiled(const float2* __restrict__ x, int64_t n, const double2* __restrict__ h, int m,
                                                                 int64_t offset, int64_t out_len, float2* __restrict__ y) {
    extern __shared__ double2 s_conv[];
    double2* s_h = s_conv;            // [m]
    double2* s_x = s_conv + m;        // [CONV_TILE + m - 1]: s_x[i] = x[first + i], zero outside the array
    for (int j = threadIdx.x; j < m; j += CONV_THREADS) s_h[j] = h[j];
    const int span = CONV_TILE + m - 1;
    for (int64_t k0 = (int64_t)blockIdx.x * CONV_TILE; k0 < out_len; k0 += (int64_t)gridDim.x * CONV_TILE) {
        const int64_t first = k0 + offset - (m - 1);   // input index of s_x[0]
        __syncthreads();                                // the previous tile's readers are done
        for (int i = threadIdx.x; i < span; i += CONV_THREADS) {
            const int64_t g = first + i;
            double2 v = make_double2(0.0, 0.0);
            if (g >= 0 && g < n) { const float2 f = x[g]; v = make_double2((double)f.x, (double)f.y); }
            s_x[i] = v;
        }
        __syncthreads();
        // output o (tile-relative) at tap j reads input index (k0 + o + offset) - j = first + (o + m - 1 - j)
        const int o0 = threadIdx.x * CONV_PER;
        double2 w[CONV_PER];   // w[i] = s_x[o0 + i + m - 1 - j]
#pragma unroll
        for (int i = 0; i < CONV_PER; i++) w[i] = s_x[o0 + i + m - 1];
        double re[CONV_PER], im[CONV_PER];
#pragma unroll
        for (int i = 0; i < CONV_PER; i++) { re[i] = 0.0; im[i] = 0.0; }
        for (int j = 0; j < m; j++) {
            const double2 c = s_h[j];
#pragma unroll
            for (int i = 0; i < CONV_PER; i++) {
                re[i] = fma(w[i].x, c.x, re[i]);
                re[i] = fma(-w[i].y, c.y, re[i]);
                im[i] = fma(w[i].x, c.y, im[i]);
                im[i] = fma(w[i].y, c.x, im[i]);
            }
            // slide the window one input sample down
#pragma unroll
            for (int i = CONV_PER - 1; i > 0; i--) w[i] = w[i - 1];
            if (j + 1 < m) w[0] = s_x[o0 + m - 2 - j];
        }
#pragma unroll
        for (int i = 0; i < CONV_PER; i++) {
            const int64_t k = k0 + o0 + i;
            if (k < out_len) y[k] = make_float2((float)re[i], (float)im[i]);
        }
    }
}

extern "C" int urh_convolve_c128(urh_ctx* ctx, const float* d_x, int64_t n, const double* d_taps, int m, int64_t offset,
                                 int64_t out_len, float* d_y) {
    if (out_len <= 0) return URH_OK;
    if (m >= 1 && m <= CONV_MAX_TAPS) {
        const size_t smem = (size_t)(m + CONV_TILE + m - 1) * sizeof(double2);   // <= 44.5 KB for m <= 768
        const unsigned grid = (unsigned)min(urh_div_up(out_len, CONV_TILE), (int64_t)ctx->sm_count * 8);
        URH_LAUNCH(ctx, k_conv_c128_tiled, grid, CONV_THREADS, smem, (const float2*)d_x, n, (const double2*)d_taps, m, offset, out_len, (float2*)d_y);
        return URH_OK;
    }
    const unsigned grid = (unsigned)min(urh_div_up(out_len, 256), (int64_t)ctx->sm_count * 32);
    URH_LAUNCH(ctx, k_conv_c128, grid, 256, 0, (const float2*)d_x, n, (const double2*)d_taps, m, offset, out_len, (float2*)d_y);
    return URH_OK;
}

// ---- the FFT branch of the band-pass and fft_convolve_1d (Filter.py:69-82): the reference transforms the whole capture, so one
// non-finite sample makes every output NaN + NaN j.  The direct convolution above leaves that to the outputs that read the sample.
// Every sample feeds at least one output of the centred crop, and with finite taps an output that reads a non-finite sample is not
// finite, so the caller flags the OUTPUTS and fills them all when one is not finite (DESIGN.md §4.5).
// *flag = 1 if any of the count floats is NaN or infinite (never cleared here, so that a flag can be carried over several calls)
__global__ void k_nonfinite_flag(const float* __restrict__ x, int64_t count, int* __restrict__ flag) {
    bool bad = false;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) bad |= !isfinite(x[i]);
    if (__syncthreads_or(bad) && threadIdx.x == 0) *flag = 1;
}

__global__ void k_nan_fill_if(float* __restrict__ y, int64_t count, const int* __restrict__ flag) {
    if (!*flag) return;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) y[i] = __int_as_float(0x7fc00000);
}

extern "C" int urh_nonfinite_flag(urh_ctx* ctx, const float* d_x, int64_t n, int* d_flag) {
    if (n <= 0) return URH_OK;
    const unsigned grid = (unsigned)min(urh_div_up(2 * n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_nonfinite_flag, grid, 256, 0, d_x, 2 * n, d_flag);
    return URH_OK;
}

extern "C" int urh_nan_fill_if(urh_ctx* ctx, float* d_y, int64_t n, const int* d_flag) {
    if (n <= 0) return URH_OK;
    const unsigned grid = (unsigned)min(urh_div_up(2 * n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_nan_fill_if, grid, 256, 0, d_y, 2 * n, d_flag);
    return URH_OK;
}

// ---- DC correction: x - mean(x, axis=0) (Filter.py:32-33) --------------------------------------------------------------
// numpy's np.mean over axis 0 of a C-contiguous float32 (n,2) array accumulates each column naively in float32 in
// row order (SURVEY H9).  exact != 0 reproduces that serial chain (one lane per column, the warp streams the data
// through shared memory); exact == 0 uses a double reduction (accurate, NOT what the reference computes for large n).
// The serial chain of one warp: lane 0 returns acc + x[0].I + x[1].I + ... (each add rounded), lane 1 the same for Q; lanes 2..31
// stream the next 1024-row chunk into shared memory meanwhile.
__device__ __forceinline__ float dc_serial_chain(const float2* __restrict__ x, int64_t n, float acc) {
    __shared__ float2 buf[2][1024];
    const int lane = threadIdx.x;
    const int64_t nchunks = (n + 1023) / 1024;
    for (int j = lane; j < 1024; j += 32) buf[0][j] = (j < n) ? x[j] : make_float2(0.f, 0.f);
    __syncwarp();
    for (int64_t c = 0; c < nchunks; c++) {
        const int b = (int)(c & 1);
        const int len = (int)min((int64_t)1024, n - c * 1024);
        if (lane < 2) {
            const float* col = (const float*)buf[b] + lane;
            for (int j = 0; j < len; j++) acc = __fadd_rn(acc, col[2 * j]);
        } else if (c + 1 < nchunks) {
            for (int j = lane - 2; j < 1024; j += 30) {
                const int64_t i = (c + 1) * 1024 + j;
                buf[b ^ 1][j] = (i < n) ? x[i] : make_float2(0.f, 0.f);
            }
        }
        __syncwarp();
    }
    return acc;
}

__global__ void __launch_bounds__(32) k_dc_mean_serial(const float2* __restrict__ x, int64_t n, float* __restrict__ mean) {
    const float acc = dc_serial_chain(x, n, 0.0f);   // lane 0: I column, lane 1: Q column
    if (threadIdx.x < 2) mean[threadIdx.x] = __fdiv_rn(acc, (float)n);  // np.mean: sum / count in float32
}

// the same chain continued from the accumulators (carry0, carry1) of the rows before x, returned undivided
__global__ void __launch_bounds__(32) k_dc_sum_serial(const float2* __restrict__ x, int64_t n, float carry0, float carry1,
                                                      double* __restrict__ sums) {
    const float acc = dc_serial_chain(x, n, threadIdx.x == 0 ? carry0 : carry1);
    if (threadIdx.x < 2) sums[threadIdx.x] = (double)acc;
}

__global__ void k_dc_mean_partial(const float2* __restrict__ x, int64_t n, double* __restrict__ part) {
    double sr = 0.0, si = 0.0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float2 v = x[i];
        sr += v.x; si += v.y;
    }
    __shared__ double s_r[256], s_i[256];
    s_r[threadIdx.x] = sr; s_i[threadIdx.x] = si;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) { s_r[threadIdx.x] += s_r[threadIdx.x + off]; s_i[threadIdx.x] += s_i[threadIdx.x + off]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { part[2 * blockIdx.x] = s_r[0]; part[2 * blockIdx.x + 1] = s_i[0]; }
}
__global__ void k_dc_mean_fold(const double* __restrict__ part, int nblocks, int64_t n, float* __restrict__ mean) {
    if (threadIdx.x < 2) {
        double s = 0.0;
        for (int b = 0; b < nblocks; b++) s += part[2 * b + threadIdx.x];
        mean[threadIdx.x] = (float)(s / (double)n);
    }
}
__global__ void k_dc_sum_fold(const double* __restrict__ part, int nblocks, double* __restrict__ sums) {
    if (threadIdx.x < 2) {
        double s = 0.0;
        for (int b = 0; b < nblocks; b++) s += part[2 * b + threadIdx.x];
        sums[threadIdx.x] = s;
    }
}
__global__ void k_dc_subtract(const float2* __restrict__ x, int64_t n, const float* __restrict__ mean, float2* __restrict__ y) {
    const float mr = mean[0], mi = mean[1];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float2 v = x[i];
        y[i] = make_float2(__fsub_rn(v.x, mr), __fsub_rn(v.y, mi));
    }
}

extern "C" int urh_dc_correction(urh_ctx* ctx, const float* d_iq, int64_t n, float* d_out, int exact_order) {
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    float* mean;
    URH_CHECK(urh_arena(ctx, 4, &mean));
    if (exact_order) {
        URH_LAUNCH(ctx, k_dc_mean_serial, 1, 32, 0, (const float2*)d_iq, n, mean);
    } else {
        const int nb = ctx->sm_count * 4;
        double* part;
        URH_CHECK(urh_arena(ctx, (size_t)nb * 2, &part));
        URH_LAUNCH(ctx, k_dc_mean_partial, nb, 256, 0, (const float2*)d_iq, n, part);
        URH_LAUNCH(ctx, k_dc_mean_fold, 1, 32, 0, part, nb, n, mean);
    }
    const unsigned grid = (unsigned)min(urh_div_up(n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_dc_subtract, grid, 256, 0, (const float2*)d_iq, n, mean, (float2*)d_out);
    return URH_OK;
}

// ---- DC correction in two steps, for a capture cut into shards: the column sums of each shard, then the subtraction of the global
// mean.  exact_order != 0: the serial float32 chain of k_dc_mean_serial continued from h_carry (NULL: from 0), so that shards handed
// over in row order reproduce urh_dc_correction's chain bit for bit; otherwise the double sums of k_dc_mean_partial / fold (the same
// grid as urh_dc_correction).  h_sums: two host doubles, not divided by anything.
extern "C" int urh_dc_column_sums(urh_ctx* ctx, const float* d_iq, int64_t n, int exact_order, const float* h_carry, double* h_sums) {
    const float c0 = h_carry ? h_carry[0] : 0.0f, c1 = h_carry ? h_carry[1] : 0.0f;
    if (n <= 0) {
        h_sums[0] = exact_order ? (double)c0 : 0.0;
        h_sums[1] = exact_order ? (double)c1 : 0.0;
        return URH_OK;
    }
    urh_arena_reset(ctx);
    double* sums;
    URH_CHECK(urh_arena(ctx, 2, &sums));
    if (exact_order) {
        URH_LAUNCH(ctx, k_dc_sum_serial, 1, 32, 0, (const float2*)d_iq, n, c0, c1, sums);
    } else {
        const int nb = ctx->sm_count * 4;
        double* part;
        URH_CHECK(urh_arena(ctx, (size_t)nb * 2, &part));
        URH_LAUNCH(ctx, k_dc_mean_partial, nb, 256, 0, (const float2*)d_iq, n, part);
        URH_LAUNCH(ctx, k_dc_sum_fold, 1, 32, 0, part, nb, sums);
    }
    URH_CUDA(ctx, cudaMemcpyAsync(h_sums, sums, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// d_out = d_iq - (mean_i, mean_q), every subtraction rounded to float32 (k_dc_subtract)
extern "C" int urh_dc_subtract(urh_ctx* ctx, const float* d_iq, int64_t n, float mean_i, float mean_q, float* d_out) {
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    float* mean;
    URH_CHECK(urh_arena(ctx, 2, &mean));
    const float h_mean[2] = {mean_i, mean_q};
    URH_CUDA(ctx, cudaMemcpyAsync(mean, h_mean, sizeof(h_mean), cudaMemcpyHostToDevice, ctx->stream));
    const unsigned grid = (unsigned)min(urh_div_up(n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_dc_subtract, grid, 256, 0, (const float2*)d_iq, n, (const float*)mean, (float2*)d_out);
    return URH_OK;
}

// ---- DC correction of an INTEGER capture: numpy promotes `x - np.mean(x, axis=0)` to float64; the column sums of integers
// are exact (int64 here, float64 pairwise in numpy: both exact below 2^53), mean = sum / n in double, result double[n][2].
template <typename T>
__global__ void __launch_bounds__(256) k_dc_int_partial(const T* __restrict__ x, int64_t n, long long* __restrict__ part) {
    long long sr = 0, si = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        sr += (long long)x[2 * i];
        si += (long long)x[2 * i + 1];
    }
    __shared__ long long s_r[256], s_i[256];
    s_r[threadIdx.x] = sr; s_i[threadIdx.x] = si;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) { s_r[threadIdx.x] += s_r[threadIdx.x + off]; s_i[threadIdx.x] += s_i[threadIdx.x + off]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { part[2 * blockIdx.x] = s_r[0]; part[2 * blockIdx.x + 1] = s_i[0]; }
}
__global__ void k_dc_int_fold(const long long* __restrict__ part, int nblocks, int64_t n, double* __restrict__ mean) {
    if (threadIdx.x < 2) {
        long long s = 0;
        for (int b = 0; b < nblocks; b++) s += part[2 * b + threadIdx.x];
        mean[threadIdx.x] = __ddiv_rn((double)s, (double)n);
    }
}
__global__ void k_dc_int_sum_fold(const long long* __restrict__ part, int nblocks, long long* __restrict__ sums) {
    if (threadIdx.x < 2) {
        long long s = 0;
        for (int b = 0; b < nblocks; b++) s += part[2 * b + threadIdx.x];
        sums[threadIdx.x] = s;
    }
}
template <typename T>
__global__ void k_dc_int_subtract(const T* __restrict__ x, int64_t n, const double* __restrict__ mean, double* __restrict__ y) {
    const double mr = mean[0], mi = mean[1];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        y[2 * i] = __dsub_rn((double)x[2 * i], mr);
        y[2 * i + 1] = __dsub_rn((double)x[2 * i + 1], mi);
    }
}

template <typename T>
static int dc_int(urh_ctx* ctx, const void* d_iq, int64_t n, double* d_out) {
    const int nb = ctx->sm_count * 4;
    long long* part;
    double* mean;
    URH_CHECK(urh_arena(ctx, (size_t)nb * 2, &part));
    URH_CHECK(urh_arena(ctx, 2, &mean));
    URH_LAUNCH(ctx, k_dc_int_partial<T>, nb, 256, 0, (const T*)d_iq, n, part);
    URH_LAUNCH(ctx, k_dc_int_fold, 1, 32, 0, (const long long*)part, nb, n, mean);
    const unsigned grid = (unsigned)min(urh_div_up(n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_dc_int_subtract<T>, grid, 256, 0, (const T*)d_iq, n, (const double*)mean, d_out);
    return URH_OK;
}

// Integer captures in two steps: exact int64 column sums of a shard (h_sums: two host int64), then d_out = d_iq - mean in double.
// Integer sums are exact, so the sums of the shards add up to the whole capture's sums in any order.
template <typename T>
static int dc_int_sums(urh_ctx* ctx, const void* d_iq, int64_t n, long long* h_sums) {
    const int nb = ctx->sm_count * 4;
    long long* part;
    long long* sums;
    URH_CHECK(urh_arena(ctx, (size_t)nb * 2, &part));
    URH_CHECK(urh_arena(ctx, 2, &sums));
    URH_LAUNCH(ctx, k_dc_int_partial<T>, nb, 256, 0, (const T*)d_iq, n, part);
    URH_LAUNCH(ctx, k_dc_int_sum_fold, 1, 32, 0, (const long long*)part, nb, sums);
    URH_CUDA(ctx, cudaMemcpyAsync(h_sums, sums, 2 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}
template <typename T>
static int dc_int_apply(urh_ctx* ctx, const void* d_iq, int64_t n, double mean_i, double mean_q, double* d_out) {
    double* mean;
    URH_CHECK(urh_arena(ctx, 2, &mean));
    const double h_mean[2] = {mean_i, mean_q};
    URH_CUDA(ctx, cudaMemcpyAsync(mean, h_mean, sizeof(h_mean), cudaMemcpyHostToDevice, ctx->stream));
    const unsigned grid = (unsigned)min(urh_div_up(n, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_dc_int_subtract<T>, grid, 256, 0, (const T*)d_iq, n, (const double*)mean, d_out);
    return URH_OK;
}

extern "C" int urh_dc_int_column_sums(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int64_t* h_sums) {
    h_sums[0] = h_sums[1] = 0;
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    long long* out = (long long*)h_sums;
    switch (dtype) {
        case URH_DT_I8: return dc_int_sums<int8_t>(ctx, d_iq, n, out);
        case URH_DT_U8: return dc_int_sums<uint8_t>(ctx, d_iq, n, out);
        case URH_DT_I16: return dc_int_sums<int16_t>(ctx, d_iq, n, out);
        case URH_DT_U16: return dc_int_sums<uint16_t>(ctx, d_iq, n, out);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "urh_dc_int_column_sums: integer capture expected");
    }
}

extern "C" int urh_dc_int_subtract(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double mean_i, double mean_q, double* d_out) {
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    switch (dtype) {
        case URH_DT_I8: return dc_int_apply<int8_t>(ctx, d_iq, n, mean_i, mean_q, d_out);
        case URH_DT_U8: return dc_int_apply<uint8_t>(ctx, d_iq, n, mean_i, mean_q, d_out);
        case URH_DT_I16: return dc_int_apply<int16_t>(ctx, d_iq, n, mean_i, mean_q, d_out);
        case URH_DT_U16: return dc_int_apply<uint16_t>(ctx, d_iq, n, mean_i, mean_q, d_out);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "urh_dc_int_subtract: integer capture expected");
    }
}

extern "C" int urh_dc_correction_int(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double* d_out) {
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    switch (dtype) {
        case URH_DT_I8: return dc_int<int8_t>(ctx, d_iq, n, d_out);
        case URH_DT_U8: return dc_int<uint8_t>(ctx, d_iq, n, d_out);
        case URH_DT_I16: return dc_int<int16_t>(ctx, d_iq, n, d_out);
        case URH_DT_U16: return dc_int<uint16_t>(ctx, d_iq, n, d_out);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "urh_dc_correction_int: integer capture expected");
    }
}

// ---- host captures of any size through the windowed ring (stream_ring.cuh, DESIGN.md §4.11) ------------------------------------------
// Each chunk runs the per-window call the sharded filters run (dist.py), on the window urh_filter_windows gives it, so its outputs are
// the resident call's words.
extern "C" int urh_convolve_c128_stream(urh_ctx* ctx, const float* h_x, int64_t n, const double* h_taps, int m, int64_t offset,
                                        int64_t out_len, int64_t chunk_samples, int ring, float* h_y) {
    if (!h_x || !h_taps || !h_y || m < 1 || offset < 0 || out_len < 0) URH_FAIL(ctx, URH_ERR_INVALID, "convolve_c128_stream: bad arguments");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_CONVOLVE, n, out_len, m, offset, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_CONVOLVE, n, out_len, URH_DT_F32, m, offset, 0, chunk_samples, L));
    const double* d_taps = (const double*)L.extra;
    URH_CUDA(ctx, cudaMemcpyAsync(L.extra, h_taps, (size_t)m * 16, cudaMemcpyHostToDevice, ctx->stream));
    return stream_run(ctx, win, R, (const char*)h_x, 8, L.in, L.z.in_slot, true,
                      [&](int64_t, const UrhWindow& w, int s) {
                          return urh_convolve_c128(ctx, (const float*)(L.in + s * L.z.in_slot), w.b - w.a, d_taps, m,
                                                   w.k0 + offset - w.a, w.k1 - w.k0, (float*)(L.out + s * L.z.out_slot));
                      },
                      contiguous_download(ctx, L.out, L.z.out_slot, (char*)h_y, 8));
}

extern "C" int urh_fir_filter_stream(urh_ctx* ctx, const float* h_x, int64_t n, const float* h_taps, int m, int64_t chunk_samples, int ring,
                                     float* h_y) {
    if (!h_x || !h_y || m < 0 || (m > 0 && !h_taps)) URH_FAIL(ctx, URH_ERR_INVALID, "fir_filter_stream: bad arguments");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_FIR, n, n, m, 0, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_FIR, n, n, URH_DT_F32, m, 0, 0, chunk_samples, L));
    const float* d_taps = (const float*)L.extra;
    if (m > 0) URH_CUDA(ctx, cudaMemcpyAsync(L.extra, h_taps, (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
    return stream_run(ctx, win, R, (const char*)h_x, 8, L.in, L.z.in_slot, true,
                      [&](int64_t, const UrhWindow& w, int s) {
                          // the slot starts at the first history sample: the chunk's own samples follow k0 - a samples in
                          const float* x = (const float*)(L.in + s * L.z.in_slot + (w.k0 - w.a) * 8);
                          return urh_fir_filter_shard(ctx, x, w.k1 - w.k0, w.k0 > 0, d_taps, m, (float*)(L.out + s * L.z.out_slot));
                      },
                      contiguous_download(ctx, L.out, L.z.out_slot, (char*)h_y, 8));
}

// Two passes: the column sums chunk by chunk (upload only), then the subtraction of the mean (upload, compute, download).  Both cut
// the capture into the same chunks, so urh_stream_stats' chunk count (set by each pass) is that number; one ring serves both, so its
// free-memory low point and arena peak cover the whole call.
//   float32, exact_order != 0: numpy's serial float32 chain continued from chunk to chunk (bit for bit urh_dc_correction);
//   float32, exact_order == 0: each chunk's double sums added in chunk order (dist.py dc_fold_double's rule), mean = float32(sum / n);
//   integer: exact int64 sums, mean = sum / n in double, float64 output (bit for bit urh_dc_correction_int).
extern "C" int urh_dc_correction_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, int exact_order, int64_t chunk_samples, int ring,
                                        void* h_out) {
    if (!h_iq || !h_out) URH_FAIL(ctx, URH_ERR_INVALID, "dc_correction_stream: bad arguments");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "dc_correction_stream: unknown dtype");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    if (n == 0) return URH_OK;
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_DC, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_DC, n, n, dtype, 0, 0, 0, chunk_samples, L));
    const int ib = urh_iq_bytes(dtype);
    const bool f32 = dtype == URH_DT_F32;
    float carry[2] = {0.0f, 0.0f};
    double dsum[2] = {0.0, 0.0};
    long long isum[2] = {0, 0};
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, ib, L.in, L.z.in_slot, false,
                         [&](int64_t, const UrhWindow& w, int s) {
                             const void* x = L.in + s * L.z.in_slot;
                             if (!f32) {
                                 int64_t part[2];
                                 URH_CHECK(urh_dc_int_column_sums(ctx, x, dtype, w.b - w.a, part));
                                 isum[0] += part[0];
                                 isum[1] += part[1];
                                 return URH_OK;
                             }
                             double part[2];
                             URH_CHECK(urh_dc_column_sums(ctx, (const float*)x, w.b - w.a, exact_order, exact_order ? carry : nullptr, part));
                             if (exact_order) {   // float32 accumulators carried in doubles: exact
                                 carry[0] = (float)part[0];
                                 carry[1] = (float)part[1];
                             } else {
                                 dsum[0] += part[0];
                                 dsum[1] += part[1];
                             }
                             return URH_OK;
                         },
                         no_download));
    float mean32[2];
    double mean64[2];
    if (f32 && exact_order) {
        mean32[0] = carry[0] / (float)n;   // np.mean: sum / count in float32 (k_dc_mean_serial)
        mean32[1] = carry[1] / (float)n;
    } else if (f32) {
        mean32[0] = (float)(dsum[0] / (double)n);
        mean32[1] = (float)(dsum[1] / (double)n);
    } else {
        mean64[0] = (double)isum[0] / (double)n;
        mean64[1] = (double)isum[1] / (double)n;
    }
    const int64_t ob = f32 ? 8 : 16;
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, ib, L.in, L.z.in_slot, true,
                         [&](int64_t, const UrhWindow& w, int s) {
                             const void* x = L.in + s * L.z.in_slot;
                             void* y = L.out + s * L.z.out_slot;
                             if (f32) return urh_dc_subtract(ctx, (const float*)x, w.b - w.a, mean32[0], mean32[1], (float*)y);
                             return urh_dc_int_subtract(ctx, x, dtype, w.b - w.a, mean64[0], mean64[1], (double*)y);
                         },
                         contiguous_download(ctx, L.out, L.z.out_slot, (char*)h_out, ob)));
    return URH_OK;
}
