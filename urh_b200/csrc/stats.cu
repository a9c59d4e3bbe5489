// Auto-interpretation statistics on the GPU (SURVEY §8a rows a5-a8):
//   magnitudes / noise level  — util.get_magnitudes (util.pyx:128-136), AutoInterpretation.detect_noise_level (:60-91)
//   center detection          — AutoInterpretation.detect_center (:226-277): rank trimming, min/max/var, histogram
//   message segmentation      — auto_interpretation.segment_messages_from_magnitudes (auto_interpretation.pyx:55-111)
//   plateau lengths           — auto_interpretation.get_plateau_lengths (:179-208)
//   median filter, dB         — auto_interpretation.median_filter (:211-240), util.arr2decibel (util.pyx:38-48)
// Host captures too large for the device: the noise level (AutoInterpretation.py:60-104) and the segmentation of estimate()
// (AutoInterpretation.py:373-471 over auto_interpretation.pyx:55-111) also stream through the rings of stream_ring.cuh, bit-identical.
// The small, data-dependent decision logic (which chunks are quiet, which histogram bins are local maxima)
// stays on the host in urh_b200/ainterpretation/AutoInterpretation.py, exactly as in the reference; the
// sample-rate reductions run here.
#include "dense_f32.cuh"
#include "sparse.cuh"
#include "stream_ring.cuh"

#include <math.h>

#include <vector>

// ---- magnitudes ------------------------------------------------------------------------------------------
// float32 IQ: (double)sqrtf(fl(re*re + im*im)); integer IQ: squares and sum in (wrapping) int32, double sqrt.
template <int DT>
__device__ __forceinline__ double urh_magnitude(const void* iq, int64_t i) {
    typedef typename UrhElem<DT>::type E;
    const E* p = (const E*)iq + 2 * i;
    if (DT == URH_DT_F32) {
        const float re = (float)p[0], im = (float)p[1];
        return (double)__fsqrt_rn(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)));
    } else {
        const uint32_t re = (uint32_t)(int32_t)p[0], im = (uint32_t)(int32_t)p[1];
        const int32_t ssum = (int32_t)(re * re + im * im);
        return sqrt((double)ssum);
    }
}

template <int DT>
__global__ void k_magnitudes(const void* __restrict__ iq, int64_t n, double* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = urh_magnitude<DT>(iq, i);
}

#define URH_DISPATCH_DT(dtype, KERNEL_CALL)                         \
    switch (dtype) {                                                \
        case URH_DT_I8: { constexpr int DT = URH_DT_I8; KERNEL_CALL; } break;   \
        case URH_DT_U8: { constexpr int DT = URH_DT_U8; KERNEL_CALL; } break;   \
        case URH_DT_I16: { constexpr int DT = URH_DT_I16; KERNEL_CALL; } break; \
        case URH_DT_U16: { constexpr int DT = URH_DT_U16; KERNEL_CALL; } break; \
        case URH_DT_F32: { constexpr int DT = URH_DT_F32; KERNEL_CALL; } break; \
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");  \
    }

extern "C" int urh_get_magnitudes(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, double* d_out) {
    if (n <= 0) return URH_OK;
    const unsigned grid = (unsigned)min((int64_t)ctx->sm_count * 16, urh_div_up(n, 256));
    URH_DISPATCH_DT(dtype, URH_LAUNCH(ctx, k_magnitudes<DT>, grid, 256, 0, d_iq, n, d_out));
    return URH_OK;
}

// ---- chunk statistics for detect_noise_level -----------------------------------------------------------------
// Chunks are counted from the END of the array (AutoInterpretation.py:66-72): chunk j covers
// [n - (j+1)*cs, n - j*cs).  Each block reduces a slice of one chunk to (sum, max) in double; a second kernel
// folds the slices in a fixed order, so the result is deterministic.
// Block b reduces slice g0 + b in sample order (urh_filter_windows' URH_FILTER_NOISE numbering: chunk nchunks - 1 - g / 64, slice
// g % 64) into that slice's slot chunk * 64 + slice, so a streamed window of slices computes each of them as the resident launch
// (g0 = 0, every slice) does.
#define STAT_BLOCK 256
#define STAT_SLICES URH_NOISE_SLICES

template <typename LOADER>
__global__ void __launch_bounds__(STAT_BLOCK) k_chunk_partial(LOADER ld, int64_t n, int64_t cs, int nchunks, int64_t g0,
                                                              double* __restrict__ psum, double* __restrict__ pmax) {
    const int64_t g = g0 + blockIdx.x;
    const int chunk = nchunks - 1 - (int)(g / STAT_SLICES), slice = (int)(g % STAT_SLICES);
    const int64_t c0 = n - (int64_t)(chunk + 1) * cs;
    const int64_t per = urh_div_up(cs, STAT_SLICES);
    const int64_t s0 = c0 + (int64_t)slice * per;
    const int64_t s1 = min(s0 + per, c0 + cs);
    double sum = 0.0, mx = -1.0;
    for (int64_t i = s0 + threadIdx.x; i < s1; i += STAT_BLOCK) {
        const double m = ld(i);
        sum += m;
        mx = fmax(mx, m);   // NaN-ignoring like a sequence of `if e > maximum`
    }
    __shared__ double s_sum[STAT_BLOCK], s_max[STAT_BLOCK];
    s_sum[threadIdx.x] = sum;
    s_max[threadIdx.x] = mx;
    __syncthreads();
    for (int off = STAT_BLOCK / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
            s_sum[threadIdx.x] += s_sum[threadIdx.x + off];
            s_max[threadIdx.x] = fmax(s_max[threadIdx.x], s_max[threadIdx.x + off]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        psum[chunk * STAT_SLICES + slice] = s_sum[0];
        pmax[chunk * STAT_SLICES + slice] = s_max[0];
    }
}

__global__ void k_chunk_final(const double* __restrict__ psum, const double* __restrict__ pmax, int nchunks,
                              double* __restrict__ sum, double* __restrict__ mx) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    double s = 0.0, m = -1.0;
    for (int j = 0; j < STAT_SLICES; j++) {
        s += psum[c * STAT_SLICES + j];
        m = fmax(m, pmax[c * STAT_SLICES + j]);
    }
    sum[c] = s;
    mx[c] = m;
}

template <int DT>
struct LoadMagIQ {
    const void* iq;
    __device__ __forceinline__ double operator()(int64_t i) const { return urh_magnitude<DT>(iq, i); }
};
template <typename T>
struct LoadReal {
    const T* x;
    __device__ __forceinline__ double operator()(int64_t i) const { return (double)x[i]; }
};

template <typename LOADER>
static int chunk_stats(urh_ctx* ctx, LOADER ld, int64_t n, int64_t cs, int nchunks, double* h_sum, double* h_max) {
    urh_arena_reset(ctx);
    double *psum, *pmax, *sum, *mx;
    URH_CHECK(urh_arena(ctx, (size_t)nchunks * STAT_SLICES, &psum));
    URH_CHECK(urh_arena(ctx, (size_t)nchunks * STAT_SLICES, &pmax));
    URH_CHECK(urh_arena(ctx, (size_t)nchunks, &sum));
    URH_CHECK(urh_arena(ctx, (size_t)nchunks, &mx));
    URH_LAUNCH(ctx, (k_chunk_partial<LOADER>), (unsigned)(nchunks * STAT_SLICES), STAT_BLOCK, 0, ld, n, cs, nchunks, (int64_t)0, psum,
               pmax);
    URH_LAUNCH(ctx, k_chunk_final, (unsigned)urh_div_up(nchunks, 128), 128, 0, psum, pmax, nchunks, sum, mx);
    URH_CUDA(ctx, cudaMemcpyAsync(h_sum, sum, nchunks * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_max, mx, nchunks * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// per-chunk (sum, max) of the magnitudes of an IQ capture, never materialising the float64 magnitude array
extern "C" int urh_noise_chunk_stats_iq(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int64_t chunksize,
                                        int nchunks, double* h_sum, double* h_max) {
    if (nchunks <= 0 || chunksize <= 0 || (int64_t)nchunks * chunksize > n) URH_FAIL(ctx, URH_ERR_INVALID, "bad chunking");
    URH_DISPATCH_DT(dtype, { LoadMagIQ<DT> ld; ld.iq = d_iq; URH_CHECK(chunk_stats(ctx, ld, n, chunksize, nchunks, h_sum, h_max)); });
    return URH_OK;
}

// The same from a host capture of any size through the windowed ring (stream_ring.cuh): each window of whole slices
// (urh_filter_windows, URH_FILTER_NOISE) is uploaded into its slot and reduced by k_chunk_partial through a pointer shifted back by
// the window's first sample, so every slice's partial is the resident launch's word; the head before n - nchunks * cs is never read.
template <int DT>
static int noise_stream(urh_ctx* ctx, const void* h_iq, int64_t n, int64_t cs, int nchunks, int64_t chunk_samples, int ring,
                        double* h_sum, double* h_max) {
    urh_arena_reset(ctx);   // the call takes no arena: its peak (urh_stream_stats) is 0, not a previous call's
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_NOISE, n, 0, cs, nchunks, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_NOISE, n, 0, DT, cs, nchunks, 0, chunk_samples, L));
    const int64_t G = (int64_t)nchunks * STAT_SLICES;
    double* psum = (double*)L.extra;
    double* pmax = (double*)(L.extra + r256(G * 8));
    double* sum = (double*)(L.extra + 2 * r256(G * 8));
    double* mx = (double*)(L.extra + 2 * r256(G * 8) + r256((int64_t)nchunks * 8));
    const int ib = urh_iq_bytes(DT);
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, ib, L.in, L.z.in_slot, false,
                         [&](int64_t, const UrhWindow& w, int s) {
                             LoadMagIQ<DT> ld;
                             ld.iq = L.in + s * L.z.in_slot - w.a * ib;   // sample i of the capture at ld.iq + i
                             URH_LAUNCH(ctx, (k_chunk_partial<LoadMagIQ<DT>>), (unsigned)(w.k1 - w.k0), STAT_BLOCK, 0, ld, n, cs,
                                        nchunks, w.k0, psum, pmax);
                             return URH_OK;
                         },
                         no_download));
    URH_LAUNCH(ctx, k_chunk_final, (unsigned)urh_div_up(nchunks, 128), 128, 0, psum, pmax, nchunks, sum, mx);
    URH_CUDA(ctx, cudaMemcpyAsync(h_sum, sum, nchunks * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_max, mx, nchunks * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

extern "C" int urh_noise_chunk_stats_iq_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, int64_t chunksize, int nchunks,
                                               int64_t chunk_samples, int ring, double* h_sum, double* h_max) {
    if (!h_iq || !h_sum || !h_max) URH_FAIL(ctx, URH_ERR_INVALID, "noise_chunk_stats_iq_stream: bad arguments");
    if (nchunks <= 0 || chunksize <= 0 || (int64_t)nchunks * chunksize > n) URH_FAIL(ctx, URH_ERR_INVALID, "bad chunking");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    URH_DISPATCH_DT(dtype, URH_CHECK(noise_stream<DT>(ctx, h_iq, n, chunksize, nchunks, chunk_samples, ring, h_sum, h_max)));
    return URH_OK;
}
int urh_chunk_sums_f32(urh_ctx* ctx, const float* d_a, int64_t n, int64_t len, int batch, float* d_out);   // pairwise.cu

// the same on an existing magnitude array (float32: is_f64 = 0, float64: is_f64 = 1).  For float32 magnitudes h_sum holds
// np.mean's own float32 sum of each chunk (numpy's pairwise summation, replayed by pairwise.cu), which the caller divides in
// float32 as np.mean does: a double sum rounds differently and flips chunks on the `mean <= 1.1 * min` edge.
extern "C" int urh_noise_chunk_stats(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, int64_t chunksize, int nchunks,
                                     double* h_sum, double* h_max) {
    if (nchunks <= 0 || chunksize <= 0 || (int64_t)nchunks * chunksize > n) URH_FAIL(ctx, URH_ERR_INVALID, "bad chunking");
    if (is_f64) {
        LoadReal<double> ld; ld.x = (const double*)d_mags;
        return chunk_stats(ctx, ld, n, chunksize, nchunks, h_sum, h_max);
    }
    LoadReal<float> ld; ld.x = (const float*)d_mags;
    URH_CHECK(chunk_stats(ctx, ld, n, chunksize, nchunks, h_sum, h_max));   // the maxima (and double sums, replaced below)
    float* d_pw;
    URH_CHECK(urh_arena(ctx, (size_t)2 * nchunks, &d_pw));
    URH_CHECK(urh_chunk_sums_f32(ctx, (const float*)d_mags, n, chunksize, nchunks, d_pw));
    std::vector<float> pw((size_t)2 * nchunks);
    URH_CUDA(ctx, cudaMemcpyAsync(pw.data(), d_pw, pw.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int c = 0; c < nchunks; c++) h_sum[c] = (double)pw[2 * c];
    return URH_OK;
}

// ---- run tables for the segmenter and the plateau RLE ----------------------------------------------------------------
// SrcAbove: class = x > thr (segment_messages, tolerance 9 <=> 10 consecutive samples, auto_interpretation.pyx:69)
// SrcCenter: class = x <= thr ? 0 : 1 (get_plateau_lengths, tolerance 0: every run start)
// The dense pass of one call or chunk, its tables the first of a fresh arena.  first_above != NULL: *first_above = sample 0 > thr,
// compared in T (double for float64 magnitudes); it is read before the pass is enqueued, so the wait covers only earlier work.
template <typename SRC, typename T>
static int run_table(urh_ctx* ctx, const T* d_x, int64_t n, float thr, int tol, UrhRunTable* rt, int* first_above) {
    urh_arena_reset(ctx);
    if (first_above) {
        T x0;
        URH_CUDA(ctx, cudaMemcpyAsync(&x0, d_x, sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *first_above = (x0 > (T)thr) ? 1 : 0;
    }
    UrhClassify cls;
    memset(&cls, 0, sizeof(cls));
    cls.noise_value = 0.0f;
    cls.order = 2;
    cls.thr[0] = thr;
    const int64_t ntiles = urh_div_up(n, URH_TILE);
    rt->n = n;
    rt->tol = tol;
    rt->cap = stage_cap_for(tol);
    URH_CHECK(urh_arena(ctx, (size_t)ntiles, &rt->tiles));
    URH_CHECK(urh_arena(ctx, (size_t)ntiles * rt->cap, &rt->staging));
    const unsigned grid = (unsigned)urh_div_up(ntiles, URH_WARPS_PER_BLOCK);
    const int vec_in = (((uintptr_t)d_x % (2 * sizeof(T))) == 0) ? 1 : 0;
    URH_LAUNCH(ctx, (k_dense_f32<SRC, T>), grid, URH_WARPS_PER_BLOCK * 32, 0, d_x, n, vec_in, cls, tol, rt->tiles, rt->staging, rt->cap,
               (int16_t*)nullptr, 0);
    return URH_OK;
}

// candidates [0, count) of c in host memory (synchronises)
static int candidates_to_host(urh_ctx* ctx, const UrhCandidates& c, int64_t count, int64_t* h_pos, int16_t* h_cls) {
    if (count == 0) return URH_OK;
    URH_CUDA(ctx, cudaMemcpyAsync(h_pos, c.pos, (size_t)count * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(h_cls, c.cls, (size_t)count * sizeof(int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

// urh_collect_candidates_shard with the candidates appended to host lists (they are few); *c keeps the table's closing run
static int collect_on_host(urh_ctx* ctx, const UrhRunTable& rt, UrhShardCarry carry, int64_t global_offset, UrhCandidates* c,
                           std::vector<int64_t>& pos, std::vector<int16_t>& cls) {
    URH_CHECK(urh_collect_candidates_shard(ctx, rt, carry, global_offset, c));
    const size_t at = pos.size();
    pos.resize(at + (size_t)c->count);
    cls.resize(at + (size_t)c->count);
    return candidates_to_host(ctx, *c, c->count, pos.data() + at, cls.data() + at);
}

// The run that ends after a piece (chunk or shard) of a capture: the piece's closing run, extended by the carry (the run that ends
// right before the piece) if the piece is one whole run of the carry's class.  dist.py fold_closing_run is the same rule.
static UrhShardCarry fold_closing_run(UrhShardCarry carry, const UrhCandidates& piece) {
    if (carry.valid && piece.whole && piece.last_cls == carry.cls) {
        carry.len += piece.last_len;
    } else {
        carry.cls = piece.last_cls;
        carry.len = piece.last_len;
    }
    carry.valid = 1;
    return carry;
}

// The two-state machine of segment_messages_from_magnitudes over the run table (host; the runs of >= 10 samples are few):
// h_pos / h_cls = candidates of tolerance 9 (index of the 10th consecutive sample of a run, its class 0 = below / 1 = above the
// noise threshold), first_above = class of sample 0, (last_cls, last_len) = the run that ends the capture.  Pure host code, so the
// sharded path (urh_b200/dist.py: candidates of all shards concatenated) shares it with urh_segment_messages.
extern "C" int urh_segments_from_runs(const int64_t* h_pos, const int16_t* h_cls, int64_t count, int first_above, int last_cls,
                                      int64_t last_len, int64_t n, int64_t* h_segments, int64_t cap, int64_t* k) {
    int state = first_above ? 1 : 0;
    int64_t start = 0, m = 0;
    for (int64_t j = 0; j < count; j++) {
        if (h_cls[j] == state) continue;
        const int64_t p = h_pos[j];  // index of the 10th consecutive sample of the opposite class
        if (state == 1) {
            if (m < cap) { h_segments[2 * m] = start; h_segments[2 * m + 1] = p - 10; }
            m++;
            state = 0;
        } else {
            start = p - 10;
            state = 1;
        }
    }
    if (state == 1) {
        const int64_t conseq_below = (last_cls == 0) ? last_len : 0;
        if (start < n - conseq_below) {
            if (m < cap) { h_segments[2 * m] = start; h_segments[2 * m + 1] = n - conseq_below; }
            m++;
        }
    }
    *k = m;
    return URH_OK;
}

// the segments of a capture of n samples from all its candidates into the context (urh_fetch_segments); last = the run that ends it
static int segments_to_ctx(urh_ctx* ctx, const std::vector<int64_t>& pos, const std::vector<int16_t>& cls, int first_above,
                           UrhShardCarry last, int64_t n, int64_t* k) {
    const int64_t cap = (int64_t)pos.size() + 1;   // a message starts at sample 0 or at a candidate
    ctx->segments.resize((size_t)(2 * cap));
    URH_CHECK(urh_segments_from_runs(pos.data(), cls.data(), (int64_t)pos.size(), first_above, last.cls, last.len, n, ctx->segments.data(),
                                     cap, k));
    ctx->segments.resize((size_t)(2 * *k));
    return URH_OK;
}

// segment_messages_from_magnitudes (auto_interpretation.pyx:55-111).  d_mags float32 (is_f64=0) or float64.  *k = number of
// messages; their (start, end) pairs stay in the context for urh_fetch_segments.
extern "C" int urh_segment_messages(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, float noise_threshold, int64_t* k) {
    *k = 0;
    ctx->segments.clear();
    if (n <= 0) return URH_OK;
    UrhRunTable rt;
    int first_above = 0;
    URH_CHECK((is_f64 ? run_table<SrcAbove, double>(ctx, (const double*)d_mags, n, noise_threshold, 9, &rt, &first_above)
                      : run_table<SrcAbove, float>(ctx, (const float*)d_mags, n, noise_threshold, 9, &rt, &first_above)));
    UrhCandidates cand;
    std::vector<int64_t> pos;
    std::vector<int16_t> cls;
    URH_CHECK(collect_on_host(ctx, rt, UrhShardCarry{}, 0, &cand, pos, cls));
    return segments_to_ctx(ctx, pos, cls, first_above, fold_closing_run(UrhShardCarry{}, cand), n, k);
}

// segment_messages_from_magnitudes(get_magnitudes(iq)) of a host capture of any size (stream_run: chunks of whole tiles).  Each chunk's
// float64 magnitudes go into a scratch of one chunk; the run-table pass over them and the candidate collector, continued from the
// run that ends right before the chunk and offset to global positions, append the chunk's candidates.  The two-state machine then
// runs once over all candidates; the segments stay in the context for urh_fetch_segments, so a caller never streams the capture
// twice to size its buffer.
extern "C" int urh_segment_messages_iq_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, float noise_threshold,
                                              int64_t chunk_samples, int ring, int64_t* k) {
    if (!h_iq || !k) URH_FAIL(ctx, URH_ERR_INVALID, "segment_messages_iq_stream: bad arguments");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    if (n < 0 || ring < 2 || ring > URH_STREAM_MAX_RING) URH_FAIL(ctx, URH_ERR_INVALID, "segment_messages_iq_stream: bad n or ring");
    *k = 0;
    ctx->segments.clear();
    if (n == 0) return URH_OK;
    const SegmentStreamSizes z = urh_segment_stream_sizes(n, dtype, chunk_samples);
    StreamRing R;
    URH_CHECK(R.init(ctx, ring, ring * z.src_slot + z.mag_bytes));
    double* d_mag = (double*)(R.mem + ring * z.src_slot);
    std::vector<int64_t> pos;
    std::vector<int16_t> cls;
    int first_above = 0;
    UrhShardCarry carry{};   // the run that ends right before the chunk
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
    URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, urh_iq_bytes(dtype), R.mem, z.src_slot, false,
                         [&](int64_t c, const UrhWindow& w, int s) {
                             URH_CHECK(urh_get_magnitudes(ctx, R.mem + s * z.src_slot + URH_STREAM_PAD, dtype, w.k1 - w.k0, d_mag));
                             UrhRunTable rt;
                             URH_CHECK((run_table<SrcAbove, double>(ctx, d_mag, w.k1 - w.k0, noise_threshold, 9, &rt,
                                                                    c == 0 ? &first_above : nullptr)));
                             UrhCandidates cand;
                             URH_CHECK(collect_on_host(ctx, rt, carry, w.k0, &cand, pos, cls));
                             carry = fold_closing_run(carry, cand);
                             return URH_OK;
                         },
                         no_download, place_after_pad));
    return segments_to_ctx(ctx, pos, cls, first_above, carry, n, k);
}

// the segments of the last urh_segment_messages or urh_segment_messages_iq_stream call: (start, end) pairs
extern "C" int urh_fetch_segments(urh_ctx* ctx, int64_t* h_segments, int64_t k) {
    if (k < 0 || 2 * k > (int64_t)ctx->segments.size()) URH_FAIL(ctx, URH_ERR_INVALID, "fetch_segments: k exceeds the last result");
    if (k > 0) memcpy(h_segments, ctx->segments.data(), (size_t)(2 * k) * sizeof(int64_t));
    return URH_OK;
}

// ---- sharded message segmentation (SURVEY 8e) -----------------------------------------------------------------------------------
// urh_segment_shard_pass leaves its shard's tile table in the context; once the ranks have exchanged their closing runs,
// urh_shard_candidates turns it into the shard's candidate table with global positions and urh_fetch_candidates copies that to the
// host.  Both tables are arena memory; rt.tiles is NULL when no pass is pending.
struct UrhShardState {
    UrhRunTable rt;
    UrhCandidates cand;
};
static UrhShardState* shard_state(urh_ctx* ctx) {
    if (!ctx->shard_state) ctx->shard_state = calloc(1, sizeof(UrhShardState));
    return (UrhShardState*)ctx->shard_state;
}

// One shard of a capture whose magnitudes are spread over the ranks: the dense pass (class = above the threshold, tolerance 9).
// h_summary = {last_cls, last_len, whole, class of the shard's first sample}.
extern "C" int urh_segment_shard_pass(urh_ctx* ctx, const void* d_mags, int is_f64, int64_t n, float noise_threshold, int64_t* h_summary) {
    if (n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "empty shard");
    UrhShardState* S = shard_state(ctx);
    int first_above = 0;
    URH_CHECK((is_f64 ? run_table<SrcAbove, double>(ctx, (const double*)d_mags, n, noise_threshold, 9, &S->rt, &first_above)
                      : run_table<SrcAbove, float>(ctx, (const float*)d_mags, n, noise_threshold, 9, &S->rt, &first_above)));
    URH_CHECK(urh_shard_run_total(ctx, n, S->rt.tiles, h_summary));   // synchronises
    h_summary[3] = first_above;
    return URH_OK;
}

// After the summaries were exchanged: carry_* describe the run that ends right before this shard (fold of the preceding shards'
// summaries; carry_valid = 0 on the first shard).  Positions are global.
// *last_cand_cls = class of the shard's last candidate (meaningful when *count > 0).
extern "C" int urh_shard_candidates(urh_ctx* ctx, int carry_valid, int carry_cls, int64_t carry_len, int64_t global_offset,
                                    int64_t* count, const int64_t** d_pos, const int16_t** d_cls, int* last_cand_cls) {
    UrhShardState* S = shard_state(ctx);
    if (!S->rt.tiles) URH_FAIL(ctx, URH_ERR_INVALID, "urh_segment_shard_pass must precede urh_shard_candidates");
    URH_CHECK(urh_collect_candidates_shard(ctx, S->rt, UrhShardCarry{carry_valid, carry_cls, carry_len}, global_offset, &S->cand));
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
    S->rt.tiles = nullptr;
    return URH_OK;
}

// host copies of the candidate table urh_shard_candidates left on the device
extern "C" int urh_fetch_candidates(urh_ctx* ctx, int64_t* h_pos, int16_t* h_cls, int64_t count) {
    UrhShardState* S = shard_state(ctx);
    if (count < 0 || count > S->cand.count) URH_FAIL(ctx, URH_ERR_INVALID, "fetch_candidates: count exceeds the table");
    return candidates_to_host(ctx, S->cand, count, h_pos, h_cls);
}

// get_plateau_lengths (auto_interpretation.pyx:179-208): h_out capacity `cap`; *k = number of plateaus.
extern "C" int urh_plateau_lengths(urh_ctx* ctx, const float* d_rect, int64_t n, float center, int percentage,
                                   uint64_t* h_out, int64_t cap, int64_t* k) {
    *k = 0;
    if (n <= 0) return URH_OK;
    UrhRunTable rt;
    URH_CHECK((run_table<SrcCenter, float>(ctx, d_rect, n, center, 0, &rt, nullptr)));
    UrhCandidates cand;
    std::vector<int64_t> pos;
    std::vector<int16_t> cls;
    URH_CHECK(collect_on_host(ctx, rt, UrhShardCarry{}, 0, &cand, pos, cls));
    // candidates with tolerance 0 are the run starts (the first one is position 0)
    const uint64_t limit = (uint64_t)percentage * (uint64_t)n / 100;
    uint64_t sum = 0;
    int64_t m = 0;
    for (size_t j = 1; j < pos.size(); j++) {
        // the reference checks `current_sum >= limit` at the top of every sample iteration, i.e. before a
        // boundary at pos[j] can append the run that ends there
        if (sum >= limit) break;
        const uint64_t len = (uint64_t)(pos[j] - pos[j - 1]);
        if (m < cap) h_out[m] = len;
        m++;
        sum += len;
    }
    if (limit == 0) m = 0;
    *k = m;
    return URH_OK;
}

// ---- median filter (auto_interpretation.pyx:211-240) ---------------------------------------------------------------------
// window [i, i+k) truncated at the end; values converted to float32 first; result = sorted[k'//2]
__global__ void k_median(const double* __restrict__ x, int64_t n, int k, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float buf[64];
    int kk = k;
    if (i + kk > n) kk = (int)(n - i);
    for (int j = 0; j < kk; j++) {
        const float v = (float)x[i + j];
        int p = j;
        while (p > 0 && buf[p - 1] > v) { buf[p] = buf[p - 1]; p--; }
        buf[p] = v;
    }
    out[i] = buf[kk / 2];
}

extern "C" int urh_median_filter(urh_ctx* ctx, const double* d_x, int64_t n, unsigned int k, float* d_out) {
    if (n <= 0) return URH_OK;
    if (k == 0 || k > 64) URH_FAIL(ctx, URH_ERR_INVALID, "median_filter: k must be in 1..64");
    URH_LAUNCH(ctx, k_median, (unsigned)urh_div_up(n, 128), 128, 0, d_x, n, (int)k, d_out);
    return URH_OK;
}

// ---- arr2decibel (util.pyx:38-48): 10.0f * log10f(re*re + im*im), float32 ------------------------------------------
__global__ void k_decibel(const float2* __restrict__ x, int64_t count, float* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const float2 v = x[i];
        out[i] = __fmul_rn(10.0f, log10f(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y))));
    }
}

extern "C" int urh_arr2decibel(urh_ctx* ctx, const float* d_complex, int64_t count, float* d_out) {
    if (count <= 0) return URH_OK;
    const unsigned grid = (unsigned)min((int64_t)ctx->sm_count * 16, urh_div_up(count, 256));
    URH_LAUNCH(ctx, k_decibel, grid, 256, 0, (const float2*)d_complex, count, d_out);
    return URH_OK;
}
