// The ring of device slots that streamed calls move a host capture through (DESIGN.md §4.11), shared by the demodulation entries
// (digitize.cu), the filter and spectrogram entries (filter.cu, spectrogram.cu) and the auto-interpretation entries (stats.cu,
// convert.cu).
//
// A chunk owns the outputs [k0, k1) and uploads the input window [a, b) those outputs read, halos included, straight from host memory,
// so no chunk reads another chunk's slot.  urh_filter_windows cuts a capture into such chunks (two plans: whole tiles with at most a
// one-sample halo, URH_FILTER_TILES; the windows of the filter, spectrogram, noise and conversion entries), urh_stream_window_schedule
// orders their copies and computations (op semantics there), and stream_run issues that order.
#pragma once
#include "common.cuh"

#define URH_STREAM_MAX_RING 8
#define URH_NOISE_SLICES 64   // slices per noise chunk (stats.cu STAT_SLICES)
#define URH_STREAM_PAD 256   // tile-chunk slot = [pad][halo][chunk]: the chunk starts 256 bytes in, the halo sample right before it
#define URH_ARENA_BLOCK ((int64_t)64 << 20)   // the scratch arena grows in blocks of at least 64 MiB (context.cu urh_arena_alloc)
enum { URH_OP_UPLOAD = 0, URH_OP_COMPUTE = 1, URH_OP_DOWNLOAD = 2 };

static inline int64_t r256(int64_t b) { return (b + 255) & ~(int64_t)255; }
// device bytes the arena may take for a streamed call's requests: a request that does not fit the current block's rest opens a new
// block, so new blocks hold at most twice the requests plus one block
static inline int64_t stream_arena_bytes(int64_t requests) { return 2 * requests + URH_ARENA_BLOCK; }

// The ring of one streamed call: the block, its events, and the copy streams drained before the block is freed on every exit path.
// arena_peak: the most scratch-arena bytes live at once over every chunk stream_run computed (a chunk's computation may reset the
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

// the slots of urh_segment_messages_iq_stream (stats.cu): chunk samples, one IQ slot ([pad][chunk], 256-byte multiple), the float64
// magnitude scratch of one chunk, the arena requests of one chunk's segmenter pass (urh_stream_footprint, digitize.cu)
struct SegmentStreamSizes {
    int64_t cs, src_slot, mag_bytes, arena;
};
SegmentStreamSizes urh_segment_stream_sizes(int64_t n, int dtype, int64_t chunk_samples);

// chunk c of a streamed call: it owns outputs [k0, k1) and reads input samples [a, b) (win[4 c ..] of urh_stream_windows)
struct UrhWindow {
    int64_t k0, k1, a, b;
};

// the chunks of a streamed entry (URH_FILTER_*; urh_stream_windows without the C wrapper)
int urh_filter_windows(int entry, int64_t n, int64_t out_len, int64_t p0, int64_t p1, int64_t chunk_samples, const int64_t* h_seg_start,
                       const int64_t* h_seg_len, int nseg, std::vector<UrhWindow>& out);
// samples per chunk of the tile plan: chunk_samples (<= 0: 2^24) rounded down to whole tiles, at least one; a capture shorter than a
// chunk is one chunk of its whole tiles
int64_t stream_chunk_samples(int64_t n, int64_t chunk_samples);

// Where a chunk's window lands in its slot, in bytes from the slot's start (src_b bytes per sample): the windowed entries at the start;
// a tile chunk so that its sample k0 sits at byte URH_STREAM_PAD and its halo right before it (the IQ kernels' vector loads rely on the
// 256-byte alignment).
typedef int64_t (*UrhPlace)(const UrhWindow& w, int src_b);
static int64_t place_at_start(const UrhWindow&, int) { return 0; }
static int64_t place_after_pad(const UrhWindow& w, int src_b) { return URH_STREAM_PAD - (w.k0 - w.a) * src_b; }

// Runs the chunks win through the ring R in the order urh_stream_window_schedule gives.  h_src: host source of src_b bytes per sample;
// chunk c's window is uploaded into slot s at d_src + s * src_slot + place(w, src_b) (h_src NULL: no upload, the computation reads
// device data).  compute(c, w, s) enqueues chunk c's work on the compute stream (it may synchronise); download(c, w, s, copy_stream)
// enqueues the copies of its outputs to the host (down false: none, the computation keeps its results).  download_resident: the
// downloads read device data no later chunk rewrites, so a computation does not wait for the download before it on its slot.
// ctx->arena_peak after the run: the most over its chunks.
template <typename Compute, typename Download>
static int stream_run(urh_ctx* ctx, const std::vector<UrhWindow>& win, StreamRing& R, const char* h_src, int src_b, char* d_src,
                      int64_t src_slot, bool down, Compute&& compute, Download&& download, UrhPlace place = place_at_start,
                      bool download_resident = false) {
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
                URH_CUDA(ctx, cudaMemcpyAsync(d_src + s * src_slot + place(w, src_b), h_src + w.a * src_b, (size_t)((w.b - w.a) * src_b),
                                              cudaMemcpyHostToDevice, cp));
            URH_CUDA(ctx, cudaEventRecord(R.ev[URH_OP_UPLOAD][s], cp));
        } else if (kind == URH_OP_COMPUTE) {
            if (h_src) URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_UPLOAD][s], 0));
            if (down && !download_resident && recorded[URH_OP_DOWNLOAD][s])
                URH_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, R.ev[URH_OP_DOWNLOAD][s], 0));
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
// contiguous outputs of ob bytes each: chunk c's [k0, k1) from its output slot at d_out + s * out_slot to h_out
static auto contiguous_download(urh_ctx* ctx, const char* d_out, int64_t out_slot, char* h_out, int64_t ob) {
    return [ctx, d_out, out_slot, h_out, ob](int64_t, const UrhWindow& w, int s, cudaStream_t cp) {
        URH_CUDA(ctx, cudaMemcpyAsync(h_out + w.k0 * ob, d_out + s * out_slot, (size_t)((w.k1 - w.k0) * ob), cudaMemcpyDeviceToHost, cp));
        return URH_OK;
    };
}
// the download of a call whose chunks keep their results on the device (down false)
static int no_download(int64_t, const UrhWindow&, int, cudaStream_t) { return URH_OK; }
