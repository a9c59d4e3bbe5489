// Signal views: path_creator.create_path (path_creator.pyx:19-82) and array_to_QPath (:88-120) on the device.
//
// The min/max pass reduces the visible range [start, end) of a strided sample column to one (min, max) pair per pixel of spp
// samples.  The encoder writes the big-endian QPainterPath streams (QDataStream >> QPainterPath) of every sub-path of one call.
#include "common.cuh"

namespace {

constexpr int VIEW_WARPS = 8;          // warps per block
constexpr int64_t VIEW_ITEM = 4096;    // samples one warp reduces: a pixel is split into ceil(spp / VIEW_ITEM) items

// Order keys.  The reference walks each pixel from its head h and updates only on a strict < or >, so (h not NaN) the result is
// the first occurrence of the extreme non-NaN value and NaNs are ignored; a NaN head is both outputs.  A key maps a sample onto an
// int32 that compares like the sample: integers are their value, a float32 is its bits with the magnitude flipped when negative and
// -0 folded onto +0 (they compare equal, so the earlier one must win).  (key, index in the pixel) pairs then reduce in any order.
template <typename T>
struct ViewKey {
    static __device__ __forceinline__ bool nan(T) { return false; }
    static __device__ __forceinline__ int key(T v) { return (int)v; }
};
template <>
struct ViewKey<float> {
    static __device__ __forceinline__ bool nan(float v) { return (__float_as_uint(v) & 0x7fffffffu) > 0x7f800000u; }
    static __device__ __forceinline__ int key(float v) {
        const int b = __float_as_int(v);
        if ((b & 0x7fffffff) == 0) return 0;
        return b < 0 ? b ^ 0x7fffffff : b;
    }
};

struct MinMax {
    int kmin, kmax;
    uint32_t imin, imax;   // index of the sample in its pixel; 0xffffffff when the pixel part holds no non-NaN sample
};

__device__ __forceinline__ MinMax mm_empty() { return {INT_MAX, INT_MIN, 0xffffffffu, 0xffffffffu}; }

// b covers samples after a's, or the pair is compared by index: "right wins only if strictly smaller/larger", ties to the lower index
__device__ __forceinline__ void mm_join(MinMax& a, const MinMax& b) {
    if (b.kmin < a.kmin || (b.kmin == a.kmin && b.imin < a.imin)) { a.kmin = b.kmin; a.imin = b.imin; }
    if (b.kmax > a.kmax || (b.kmax == a.kmax && b.imax < a.imax)) { a.kmax = b.kmax; a.imax = b.imax; }
}

__device__ __forceinline__ void mm_warp(MinMax& a) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        MinMax b;
        b.kmin = __shfl_down_sync(URH_FULL_MASK, a.kmin, o);
        b.kmax = __shfl_down_sync(URH_FULL_MASK, a.kmax, o);
        b.imin = __shfl_down_sync(URH_FULL_MASK, a.imin, o);
        b.imax = __shfl_down_sync(URH_FULL_MASK, a.imax, o);
        mm_join(a, b);
    }
}

// values[2p], values[2p + 1] of pixel p starting at sample ps (relative to start); r is the whole pixel's reduction
template <typename T>
__device__ __forceinline__ void mm_store(const T* __restrict__ src, int64_t stride, int64_t start, int64_t ps, const MinMax& r,
                                         T* __restrict__ values, int64_t p) {
    const T h = src[(start + ps) * stride];
    if (ViewKey<T>::nan(h)) {
        values[2 * p] = h;
        values[2 * p + 1] = h;
    } else {
        values[2 * p] = src[(start + ps + r.imin) * stride];
        values[2 * p + 1] = src[(start + ps + r.imax) * stride];
    }
}

// One warp per item (pixel p, part c): the part's samples, lane-strided so that loads coalesce.  A pixel of one part is finished
// here; otherwise the part's reduction goes to partial[item] for k_path_fold.
template <typename T>
__global__ void __launch_bounds__(VIEW_WARPS * 32) k_path_minmax(const T* __restrict__ src, int64_t stride, int64_t start, int64_t N,
                                                                 int64_t spp, int64_t items, int64_t parts, T* __restrict__ values,
                                                                 MinMax* __restrict__ partial) {
    const int64_t item = (int64_t)blockIdx.x * VIEW_WARPS + (threadIdx.x >> 5);
    if (item >= items) return;
    const int lane = threadIdx.x & 31;
    const int64_t p = item / parts, c = item - p * parts;
    const int64_t ps = p * spp, pe = min(ps + spp, N);
    const int64_t cs = ps + c * VIEW_ITEM, ce = min(cs + VIEW_ITEM, pe);
    MinMax a = mm_empty();
    const T* base = src + start * stride;
#pragma unroll 8
    for (int64_t i = cs + lane; i < ce; i += 32) {
        const T v = base[i * stride];
        if (ViewKey<T>::nan(v)) continue;
        const int k = ViewKey<T>::key(v);
        const uint32_t rel = (uint32_t)(i - ps);
        if (k < a.kmin) { a.kmin = k; a.imin = rel; }   // a lane walks upwards: strict keeps its first occurrence
        if (k > a.kmax) { a.kmax = k; a.imax = rel; }
    }
    mm_warp(a);
    if (lane) return;
    if (parts == 1) mm_store(src, stride, start, ps, a, values, p);
    else partial[item] = a;
}

// One warp per pixel of more than one part: join its parts' reductions.
template <typename T>
__global__ void __launch_bounds__(VIEW_WARPS * 32) k_path_fold(const T* __restrict__ src, int64_t stride, int64_t start, int64_t spp,
                                                               int64_t P, int64_t parts, const MinMax* __restrict__ partial,
                                                               T* __restrict__ values) {
    const int64_t p = (int64_t)blockIdx.x * VIEW_WARPS + (threadIdx.x >> 5);
    if (p >= P) return;
    const int lane = threadIdx.x & 31;
    MinMax a = mm_empty();
    for (int64_t c = lane; c < parts; c += 32) mm_join(a, partial[p * parts + c]);
    mm_warp(a);
    if (lane == 0) mm_store(src, stride, start, p * spp, a, values, p);
}

__device__ __forceinline__ uint32_t bswap32(uint32_t w) { return __byte_perm(w, 0, 0x0123); }

// float64 bits of np.negative(v) in the sample dtype, converted to float64 as numpy does on x86 (a NaN keeps sign and payload, and
// is quieted).  Built from integer operations so that no conversion instruction decides NaN payloads or denormals.
template <typename T>
__device__ __forceinline__ uint64_t neg_f64_bits(T v) {
    return (uint64_t)__double_as_longlong((double)(T)(0 - (int)v));
}
template <>
__device__ __forceinline__ uint64_t neg_f64_bits<float>(float v) {
    const uint32_t b = __float_as_uint(v) ^ 0x80000000u;
    const uint64_t s = (uint64_t)(b >> 31) << 63;
    const uint32_t e = (b >> 23) & 0xffu, m = b & 0x7fffffu;
    if (e == 0xffu) return s | 0x7ff0000000000000ull | ((uint64_t)(m ? (m | 0x400000u) : 0u) << 29);
    if (e == 0) return s | (uint64_t)__double_as_longlong((double)m * 0x1p-149);   // zero or denormal: exact in float64
    return s | ((uint64_t)(e + 896u) << 52) | ((uint64_t)m << 29);
}

// One thread per record of every sub-path.  rec[s] is the first record of sub-path s (rec[count] = all records), lo[s] its first
// index into x / values, word[s] its first 32-bit word in out.  Stream: n, n x {1, x, y}, 0, 0, all big-endian (:102-120).
// x is x0 + (i >> 1) * spp (min/max pairs) or x0 + i; y is -values[i], or -samples[start + i] when spp <= 1.
template <typename T>
__global__ void __launch_bounds__(256) k_qpath_streams(const T* __restrict__ src, int64_t stride, int64_t start, int64_t spp,
                                                       int64_t x0, const T* __restrict__ values, const int64_t* __restrict__ rec,
                                                       const int64_t* __restrict__ lo, const int64_t* __restrict__ word, int count,
                                                       uint32_t* __restrict__ out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rec[count]) return;
    int a = 0, b = count;   // the last s with rec[s] <= r; it has r < rec[s + 1], so it is not empty
    while (b - a > 1) {
        const int m = (a + b) >> 1;
        if (rec[m] <= r) a = m;
        else b = m;
    }
    const int s = a;
    const int64_t j = r - rec[s], n = rec[s + 1] - rec[s], i = lo[s] + j;
    uint32_t* w = out + word[s];
    const int64_t xi = spp > 1 ? x0 + (i >> 1) * spp : x0 + i;
    const T y = spp > 1 ? values[i] : src[(start + i) * stride];
    const uint64_t xb = (uint64_t)__double_as_longlong((double)xi), yb = neg_f64_bits(y);
    uint32_t* q = w + 1 + 5 * j;
    q[0] = bswap32(1u);
    q[1] = bswap32((uint32_t)(xb >> 32));
    q[2] = bswap32((uint32_t)xb);
    q[3] = bswap32((uint32_t)(yb >> 32));
    q[4] = bswap32((uint32_t)yb);
    if (j == 0) w[0] = bswap32((uint32_t)n);
    if (j == n - 1) {
        w[1 + 5 * n] = 0u;
        w[2 + 5 * n] = 0u;
    }
}

template <typename T>
int path_minmax_run(urh_ctx* ctx, const T* src, int64_t stride, int64_t start, int64_t N, int64_t spp, T* values) {
    const int64_t P = urh_div_up(N, spp), parts = urh_div_up(spp, VIEW_ITEM), items = P * parts;
    MinMax* partial = nullptr;
    if (parts > 1) {
        urh_arena_reset(ctx);
        URH_CHECK(urh_arena(ctx, (size_t)items, &partial));
    }
    URH_LAUNCH(ctx, k_path_minmax<T>, (unsigned)urh_div_up(items, VIEW_WARPS), VIEW_WARPS * 32, 0, src, stride, start, N, spp, items,
               parts, values, partial);
    if (parts > 1)
        URH_LAUNCH(ctx, k_path_fold<T>, (unsigned)urh_div_up(P, VIEW_WARPS), VIEW_WARPS * 32, 0, src, stride, start, spp, P, parts,
                   partial, values);
    return URH_OK;
}

// the length of x / values: 2P min/max pairs when spp > 1, else the N samples themselves
int view_length(urh_ctx* ctx, int64_t n, int64_t start, int64_t end, int64_t spp, int64_t stride, int64_t* L) {
    if (start < 0 || end < start || end > n) URH_FAIL(ctx, URH_ERR_INVALID, "path: need 0 <= start <= end <= n (got %lld, %lld, %lld)",
                                                      (long long)start, (long long)end, (long long)n);
    if (spp < 0 || stride < 1) URH_FAIL(ctx, URH_ERR_INVALID, "path: bad samples per pixel or stride");
    if (spp >= ((int64_t)1 << 32)) URH_FAIL(ctx, URH_ERR_INVALID, "path: more than 2^32 - 1 samples per pixel");
    *L = spp > 1 ? 2 * urh_div_up(end - start, spp) : end - start;
    return URH_OK;
}

}  // namespace

extern "C" int urh_path_minmax(urh_ctx* ctx, const void* d_src, int dtype, int64_t stride, int64_t n, int64_t start, int64_t end,
                               int64_t spp, void* d_values) {
    int64_t L;
    URH_CHECK(view_length(ctx, n, start, end, spp, stride, &L));
    if (spp <= 1) URH_FAIL(ctx, URH_ERR_INVALID, "path_minmax: needs more than one sample per pixel");
    const int64_t N = end - start;
    switch (dtype) {
        case URH_DT_I8: return path_minmax_run(ctx, (const int8_t*)d_src, stride, start, N, spp, (int8_t*)d_values);
        case URH_DT_U8: return path_minmax_run(ctx, (const uint8_t*)d_src, stride, start, N, spp, (uint8_t*)d_values);
        case URH_DT_I16: return path_minmax_run(ctx, (const int16_t*)d_src, stride, start, N, spp, (int16_t*)d_values);
        case URH_DT_U16: return path_minmax_run(ctx, (const uint16_t*)d_src, stride, start, N, spp, (uint16_t*)d_values);
        case URH_DT_F32: return path_minmax_run(ctx, (const float*)d_src, stride, start, N, spp, (float*)d_values);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    }
}

extern "C" int urh_qpath_streams(urh_ctx* ctx, const void* d_src, int dtype, int64_t stride, int64_t n, int64_t start, int64_t end,
                                 int64_t spp, int64_t x0, const void* d_values, const int64_t* h_bounds, int count, uint8_t* d_out,
                                 int64_t* h_offsets) {
    int64_t L;
    URH_CHECK(view_length(ctx, n, start, end, spp, stride, &L));
    if (count < 0) URH_FAIL(ctx, URH_ERR_INVALID, "qpath_streams: negative sub-path count");
    if (dtype < URH_DT_I8 || dtype > URH_DT_F32) URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    // {rec[count + 1], lo[count], word[count]}; h_offsets[s] = byte offset of sub-path s, h_offsets[count] = total bytes
    std::vector<int64_t> tab((size_t)3 * count + 1);
    int64_t* rec = tab.data();
    int64_t *lo = rec + count + 1, *word = lo + count;
    int64_t records = 0, bytes = 0;
    for (int s = 0; s < count; s++) {
        const int64_t a = h_bounds[2 * s], b = h_bounds[2 * s + 1];
        if (a < 0 || b < 0 || a > L || b > L) URH_FAIL(ctx, URH_ERR_INVALID, "qpath_streams: sub-path %d bounds outside [0, %lld]", s, (long long)L);
        const int64_t k = b > a ? b - a : 0;
        rec[s] = records;
        lo[s] = a;
        word[s] = bytes / 4;
        h_offsets[s] = bytes;
        records += k;
        bytes += k ? 4 + 20 * k + 8 : 0;   // an empty sub-path is an empty QPainterPath(): no stream
    }
    rec[count] = records;
    h_offsets[count] = bytes;
    if (!d_out || records == 0) return URH_OK;   // size query
    if (spp > 1 && !d_values) URH_FAIL(ctx, URH_ERR_INVALID, "qpath_streams: spp > 1 needs the min/max values");
    urh_arena_reset(ctx);
    int64_t* d_tab;
    URH_CHECK(urh_arena(ctx, tab.size(), &d_tab));
    URH_CUDA(ctx, cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    const int64_t *d_rec = d_tab, *d_lo = d_tab + count + 1, *d_word = d_lo + count;
    const unsigned grid = (unsigned)urh_div_up(records, 256);
    uint32_t* out = (uint32_t*)d_out;
    switch (dtype) {
        case URH_DT_I8:
            URH_LAUNCH(ctx, k_qpath_streams<int8_t>, grid, 256, 0, (const int8_t*)d_src, stride, start, spp, x0, (const int8_t*)d_values, d_rec,
                       d_lo, d_word, count, out);
            break;
        case URH_DT_U8:
            URH_LAUNCH(ctx, k_qpath_streams<uint8_t>, grid, 256, 0, (const uint8_t*)d_src, stride, start, spp, x0, (const uint8_t*)d_values,
                       d_rec, d_lo, d_word, count, out);
            break;
        case URH_DT_I16:
            URH_LAUNCH(ctx, k_qpath_streams<int16_t>, grid, 256, 0, (const int16_t*)d_src, stride, start, spp, x0, (const int16_t*)d_values,
                       d_rec, d_lo, d_word, count, out);
            break;
        case URH_DT_U16:
            URH_LAUNCH(ctx, k_qpath_streams<uint16_t>, grid, 256, 0, (const uint16_t*)d_src, stride, start, spp, x0, (const uint16_t*)d_values,
                       d_rec, d_lo, d_word, count, out);
            break;
        default:
            URH_LAUNCH(ctx, k_qpath_streams<float>, grid, 256, 0, (const float*)d_src, stride, start, spp, x0, (const float*)d_values, d_rec,
                       d_lo, d_word, count, out);
            break;
    }
    return URH_OK;
}
