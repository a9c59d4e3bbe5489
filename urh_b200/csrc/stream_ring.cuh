// The ring of device slots that streamed calls move a host capture through (DESIGN.md §4.11), shared by the demodulation entries
// (digitize.cu) and the filter and spectrogram entries (filter.cu, spectrogram.cu).
//
// Two runners drive it:
//   stream_run          chunks of whole tiles with at most a one-sample halo; qad downloaded into h_qad (urh_stream_schedule)
//   stream_run_windows  chunks that own the outputs [k0, k1) and upload the input window [a, b) those outputs read, halos of any
//                       length included, straight from host memory; each chunk's outputs leave through a caller-given download
//                       (urh_stream_windows, urh_stream_window_schedule)
// Both issue their ops in the order their schedule lists, with the same op semantics (include/urh_b200.h).
#pragma once
#include "common.cuh"

#define URH_STREAM_MAX_RING 8
#define URH_NOISE_SLICES 64   // slices per noise chunk (stats.cu STAT_SLICES)
#define URH_STREAM_PAD 256   // slot = [pad][halo][chunk]: the chunk starts 256 bytes in, the halo sample right before it
enum { URH_OP_UPLOAD = 0, URH_OP_COMPUTE = 1, URH_OP_DOWNLOAD = 2 };

static inline int64_t r256(int64_t b) { return (b + 255) & ~(int64_t)255; }

// The ring of one streamed call: the block, its events, and the copy streams drained before the block is freed on every exit path.
// arena_peak: the most scratch-arena bytes live at once over every chunk the runners computed (a chunk's window call may reset the
// arena, which restarts ctx->arena_peak).
struct StreamRing {
    urh_ctx* ctx = nullptr;
    char* mem = nullptr;
    cudaEvent_t ev[3][URH_STREAM_MAX_RING] = {};
    int ring = 0;
    size_t arena_peak = 0;
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

// the slots of urh_segment_messages_iq_stream (stats.cu): chunk samples, one IQ slot ([pad][chunk], 256-byte multiple), the float64
// magnitude scratch of one chunk, the arena requests of one chunk's segmenter pass (urh_stream_footprint, digitize.cu)
struct SegmentStreamSizes {
    int64_t cs, src_slot, mag_bytes, arena;
};
SegmentStreamSizes urh_segment_stream_sizes(int64_t n, int dtype, int64_t chunk_samples);

// ---- the windowed ring ---------------------------------------------------------------------------------------------------------------
// A chunk c is {k0, k1, a, b} (win[4 c ..]): it owns outputs [k0, k1) and reads input samples [a, b).  Slot s holds the window from its
// first byte: d_src + s * src_slot = sample a.  compute(c, w, s) enqueues chunk c's work on the compute stream (it may synchronise);
// download(c, w, s, copy_stream) enqueues the copies of its outputs to the host.  h_src NULL: no upload (the computation reads device
// data); down false: no download (the computation keeps its results).
struct UrhWindow {
    int64_t k0, k1, a, b;
};

// the windows of a streamed filter / spectrogram entry (URH_FILTER_*; urh_stream_windows without the C wrapper)
int urh_filter_windows(int entry, int64_t n, int64_t out_len, int64_t p0, int64_t p1, int64_t chunk_samples, const int64_t* h_seg_start,
                       const int64_t* h_seg_len, int nseg, std::vector<UrhWindow>& out);

template <typename Compute, typename Download>
static int stream_run_windows(urh_ctx* ctx, const std::vector<UrhWindow>& win, StreamRing& R, const char* h_src, int src_b, char* d_src,
                              int64_t src_slot, bool down, Compute&& compute, Download&& download) {
    const int flags = (h_src ? URH_STREAM_UPLOAD : 0) | (down ? URH_STREAM_DOWNLOAD : 0);
    const int64_t chunks = (int64_t)win.size();
    int64_t count = 0;
    URH_CHECK(urh_stream_window_schedule((const int64_t*)win.data(), chunks, R.ring, flags, nullptr, 0, &count));
    std::vector<int64_t> ops((size_t)(7 * count));
    URH_CHECK(urh_stream_window_schedule((const int64_t*)win.data(), chunks, R.ring, flags, ops.data(), count, &count));
    bool recorded[3][URH_STREAM_MAX_RING] = {};
    ctx->stream_chunks = 0;
    for (int64_t i = 0; i < count; i++) {
        const int64_t* o = &ops[(size_t)(7 * i)];
        const int kind = (int)o[0], s = (int)o[2];
        const int64_t c = o[1];
        const UrhWindow w{o[3], o[4], o[5], o[6]};
        if (kind == URH_OP_UPLOAD) {
            cudaStream_t cp = ctx->copy_stream[0];
            if (recorded[URH_OP_COMPUTE][s]) URH_CUDA(ctx, cudaStreamWaitEvent(cp, R.ev[URH_OP_COMPUTE][s], 0));
            if (w.b > w.a)
                URH_CUDA(ctx, cudaMemcpyAsync(d_src + s * src_slot, h_src + w.a * src_b, (size_t)((w.b - w.a) * src_b), cudaMemcpyHostToDevice, cp));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_UPLOAD][s], cp));
        } else if (kind == URH_OP_COMPUTE) {
            if (h_src) URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_UPLOAD][s], 0));
            if (down && recorded[URH_OP_DOWNLOAD][s]) URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_DOWNLOAD][s], 0));
            URH_CHECK(compute(c, w, s));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_COMPUTE][s], ctx->stream));
            if (ctx->arena_peak > R.arena_peak) R.arena_peak = ctx->arena_peak;
            urh_stream_sample_free(ctx);
            ctx->stream_chunks++;
        } else {
            cudaStream_t cp = ctx->copy_stream[1];
            URH_CUDA(ctx, cudaStreamWaitEvent(cp, R.ev[URH_OP_COMPUTE][s], 0));
            URH_CHECK(download(c, w, s, cp));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_DOWNLOAD][s], cp));
        }
        recorded[kind][s] = true;
    }
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream[1]));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->arena_peak = R.arena_peak;
    return URH_OK;
}

// checks shared by the windowed entries; the ring block is sized by urh_stream_filter_footprint's own formula
int urh_filter_stream_check(urh_ctx* ctx, int64_t n, int ring);
struct FilterStreamSizes {
    int64_t in_slot, out_slot;   // bytes of one input / output slot (each a multiple of 256)
    int64_t extra;               // bytes after the slots for the call's small tables (taps, window, colormap, segments)
    int64_t work;                // scratch a chunk's window call takes (arena, cuFFT, the composed image path's dB rows)
};
// p2: the colormap's entries for URH_FILTER_IMAGES (0 otherwise)
FilterStreamSizes urh_filter_stream_sizes(int entry, int64_t n, int64_t out_len, int dtype, int64_t p0, int64_t p1, int64_t p2,
                                          int64_t chunk_samples);

// The block of a windowed call: [ring input slots][ring output slots][the call's small tables (taps, window, colormap)].
struct FilterRingLayout {
    FilterStreamSizes z;
    char* in;
    char* out;
    char* extra;
};
static int filter_ring_init(urh_ctx* ctx, StreamRing& R, int ring, int entry, int64_t n, int64_t out_len, int dtype, int64_t p0, int64_t p1,
                            int64_t p2, int64_t chunk_samples, FilterRingLayout& L) {
    L.z = urh_filter_stream_sizes(entry, n, out_len, dtype, p0, p1, p2, chunk_samples);
    URH_CHECK(R.init(ctx, ring, ring * (L.z.in_slot + L.z.out_slot) + L.z.extra));
    L.in = R.mem;
    L.out = R.mem + ring * L.z.in_slot;
    L.extra = L.out + ring * L.z.out_slot;
    return URH_OK;
}
// contiguous outputs of ob bytes each: chunk c's [k0, k1) from its output slot to h_out
static auto contiguous_download(urh_ctx* ctx, const FilterRingLayout& L, char* h_out, int64_t ob) {
    return [ctx, &L, h_out, ob](int64_t, const UrhWindow& w, int s, cudaStream_t cp) {
        URH_CUDA(ctx, cudaMemcpyAsync(h_out + w.k0 * ob, L.out + s * L.z.out_slot, (size_t)((w.k1 - w.k0) * ob), cudaMemcpyDeviceToHost, cp));
        return URH_OK;
    };
}
