// Sample-format conversions of IQArray.convert_to (IQArray.py:127-200) on the GPU (SURVEY §8f row 2): the capture formats
// cs8 / cu8 / cs16 / cu16 / float32 into each other, element by element, with numpy's integer wrap-around and C's
// float -> int truncation.  One pass, 1..4 bytes read and written per element.
#include "convert.cuh"
#include "stream_ring.cuh"

#include <type_traits>

template <typename S, typename D>
__global__ void k_convert(const S* __restrict__ in, D* __restrict__ out, int64_t count) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) out[i] = conv_one<S, D>(in[i]);
}

template <typename S>
static int convert_from(urh_ctx* ctx, const void* d_in, void* d_out, int out_dtype, int64_t count, unsigned grid) {
    switch (out_dtype) {
        case URH_DT_I8: if constexpr (!std::is_same<S, int8_t>::value) { URH_LAUNCH(ctx, (k_convert<S, int8_t>), grid, 256, 0, (const S*)d_in, (int8_t*)d_out, count); return URH_OK; } break;
        case URH_DT_U8: if constexpr (!std::is_same<S, uint8_t>::value) { URH_LAUNCH(ctx, (k_convert<S, uint8_t>), grid, 256, 0, (const S*)d_in, (uint8_t*)d_out, count); return URH_OK; } break;
        case URH_DT_I16: if constexpr (!std::is_same<S, int16_t>::value) { URH_LAUNCH(ctx, (k_convert<S, int16_t>), grid, 256, 0, (const S*)d_in, (int16_t*)d_out, count); return URH_OK; } break;
        case URH_DT_U16: if constexpr (!std::is_same<S, uint16_t>::value) { URH_LAUNCH(ctx, (k_convert<S, uint16_t>), grid, 256, 0, (const S*)d_in, (uint16_t*)d_out, count); return URH_OK; } break;
        case URH_DT_F32: if constexpr (!std::is_same<S, float>::value) { URH_LAUNCH(ctx, (k_convert<S, float>), grid, 256, 0, (const S*)d_in, (float*)d_out, count); return URH_OK; } break;
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Data type not supported");
    }
    // same type: plain copy
    URH_CUDA(ctx, cudaMemcpyAsync(d_out, d_in, (size_t)count * sizeof(S), cudaMemcpyDeviceToDevice, ctx->stream));
    return URH_OK;
}

// count = number of ELEMENTS (2 per IQ sample).  Asynchronous on the context's stream.
extern "C" int urh_convert_iq(urh_ctx* ctx, const void* d_in, int in_dtype, void* d_out, int out_dtype, int64_t count) {
    if (count <= 0) return URH_OK;
    const unsigned grid = (unsigned)min(urh_div_up(count, 256), (int64_t)ctx->sm_count * 32);
    switch (in_dtype) {
        case URH_DT_I8: return convert_from<int8_t>(ctx, d_in, d_out, out_dtype, count, grid);
        case URH_DT_U8: return convert_from<uint8_t>(ctx, d_in, d_out, out_dtype, count, grid);
        case URH_DT_I16: return convert_from<int16_t>(ctx, d_in, d_out, out_dtype, count, grid);
        case URH_DT_U16: return convert_from<uint16_t>(ctx, d_in, d_out, out_dtype, count, grid);
        case URH_DT_F32: return convert_from<float>(ctx, d_in, d_out, out_dtype, count, grid);
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Data type not supported");
    }
}

// The same from a host capture of any size to a host output through the windowed ring (stream_ring.cuh): chunks of whole samples
// (urh_filter_windows, URH_FILTER_CONVERT), each converted by urh_convert_iq, so every element is the resident call's.  n = samples.
extern "C" int urh_convert_iq_stream(urh_ctx* ctx, const void* h_src, int src_dtype, void* h_dst, int dst_dtype, int64_t n,
                                     int64_t chunk_samples, int ring) {
    if (!h_src || !h_dst) URH_FAIL(ctx, URH_ERR_INVALID, "convert_iq_stream: bad arguments");
    if (urh_iq_bytes(src_dtype) == 0 || urh_iq_bytes(dst_dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Data type not supported");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    if (n == 0) return URH_OK;
    urh_arena_reset(ctx);   // the call takes no arena: its peak (urh_stream_stats) is 0, not a previous call's
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(URH_FILTER_CONVERT, n, n, dst_dtype, 0, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_CONVERT, n, n, src_dtype, dst_dtype, 0, 0, chunk_samples, L));
    return stream_run(ctx, win, R, (const char*)h_src, urh_iq_bytes(src_dtype), L.in, L.z.in_slot, true,
                      [&](int64_t, const UrhWindow& w, int s) {
                          return urh_convert_iq(ctx, L.in + s * L.z.in_slot, src_dtype, L.out + s * L.z.out_slot, dst_dtype,
                                                2 * (w.k1 - w.k0));
                      },
                      contiguous_download(ctx, L.out, L.z.out_slot, (char*)h_dst, urh_iq_bytes(dst_dtype)));
}
