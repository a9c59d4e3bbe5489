// The plan of a streamed call (DESIGN.md §4.11): which outputs each chunk owns and which input window it uploads, the order of its
// copies and computations, and the device bytes of the streamed and the resident form of each windowed entry.  Host code only:
// everything here runs without a device.
#include "dense.cuh"   // URH_TILE
#include "stream_ring.cuh"

static int64_t filter_chunk(int64_t cs) { return cs > 0 ? cs : (int64_t)1 << 24; }
static int64_t frames_per_chunk(int64_t cs, int64_t hop) { return cs / hop > 0 ? cs / hop : 1; }
// frames of a segment of len samples, as Spectrogram.stft and urh_spectrogram_bgra count them (short segments: one frame)
static int64_t frames_of(int64_t len, int64_t W, int64_t hop) { return len < W ? 1 : (len - W) / hop + 1; }
static int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

int64_t stream_chunk_samples(int64_t n, int64_t cs) {
    if (cs <= 0) cs = (int64_t)1 << 24;
    cs -= cs % URH_TILE;
    if (cs < URH_TILE) cs = URH_TILE;
    const int64_t whole = urh_div_up(n > 0 ? n : 1, URH_TILE) * URH_TILE;   // a capture shorter than a chunk: one slot of its size
    return cs < whole ? cs : whole;
}

// The noise-chunk statistics (stats.cu) reduce each of the nchunks end-aligned chunks of cs samples in URH_NOISE_SLICES slices of
// ceil(cs / URH_NOISE_SLICES) samples.  Slice g in sample order is slice g % 64 of chunk nchunks - 1 - g / 64 (chunk j covers
// [n - (j + 1) cs, n - j cs)); its samples, clipped to its chunk (a slice past a short chunk's end is empty):
static void noise_slice(int64_t n, int64_t cs, int64_t nchunks, int64_t g, int64_t* s0, int64_t* s1) {
    const int64_t j = nchunks - 1 - g / URH_NOISE_SLICES, c0 = n - (j + 1) * cs, c1 = c0 + cs;
    const int64_t per = urh_div_up(cs, URH_NOISE_SLICES);
    *s0 = c0 + (g % URH_NOISE_SLICES) * per < c1 ? c0 + (g % URH_NOISE_SLICES) * per : c1;
    *s1 = *s0 + per < c1 ? *s0 + per : c1;
}
// samples of the largest noise window: a chunk, or one slice when a slice is longer, never more than the chunks cover
static int64_t noise_slot_samples(int64_t cs, int64_t nchunks, int64_t chunk_samples) {
    const int64_t per = urh_div_up(cs, URH_NOISE_SLICES);
    const int64_t w = filter_chunk(chunk_samples) > per ? filter_chunk(chunk_samples) : per;
    return w < cs * nchunks ? w : cs * nchunks;
}

int urh_filter_windows(int entry, int64_t n, int64_t out_len, int64_t p0, int64_t p1, int64_t chunk_samples, const int64_t* h_seg_start,
                       const int64_t* h_seg_len, int nseg, std::vector<UrhWindow>& out) {
    out.clear();
    if (n < 0 || out_len < 0) return URH_ERR_INVALID;
    int64_t cs = filter_chunk(chunk_samples);
    switch (entry) {
        case URH_FILTER_CONVOLVE: {   // output k reads x[k + offset - (m - 1) .. k + offset]
            const int64_t m = p0, off = p1;
            if (m < 1 || off < 0) return URH_ERR_INVALID;
            for (int64_t k0 = 0; k0 < out_len; k0 += cs) {
                const int64_t k1 = k0 + cs < out_len ? k0 + cs : out_len;
                const int64_t b = clamp64(k1 + off, 0, n);
                const int64_t a = clamp64(k0 + off - (m - 1), 0, b);
                out.push_back({k0, k1, a, b});
            }
            return URH_OK;
        }
        case URH_FILTER_FIR: {   // output k reads x[k - (m - 1) .. k]; a chunk is at least the history long
            if (p0 < 0) return URH_ERR_INVALID;
            const int64_t h = p0 > 1 ? p0 - 1 : 0;
            if (cs < h) cs = h;
            for (int64_t k0 = 0; k0 < n; k0 += cs) {
                const int64_t k1 = k0 + cs < n ? k0 + cs : n;
                out.push_back({k0, k1, k0 > 0 ? k0 - h : 0, k1});
            }
            return URH_OK;
        }
        case URH_FILTER_TILES: {   // whole tiles, so every tile keeps its resident bounds; p0 = 1: later chunks read the sample before them
            if (p0 != 0 && p0 != 1) return URH_ERR_INVALID;
            cs = stream_chunk_samples(n, chunk_samples);
            for (int64_t k0 = 0; k0 < n; k0 += cs) {
                const int64_t k1 = k0 + cs < n ? k0 + cs : n;
                out.push_back({k0, k1, k0 > 0 ? k0 - p0 : 0, k1});
            }
            return URH_OK;
        }
        case URH_FILTER_DC:
        case URH_FILTER_CONVERT:
            for (int64_t k0 = 0; k0 < n; k0 += cs) out.push_back({k0, k0 + cs < n ? k0 + cs : n, k0, k0 + cs < n ? k0 + cs : n});
            return URH_OK;
        case URH_FILTER_NOISE: {   // outputs: the slices in sample order (p0 = cs, p1 = nchunks); whole slices per window
            const int64_t ccs = p0, nchunks = p1;
            if (ccs < 1 || nchunks < 1 || ccs * nchunks > n) return URH_ERR_INVALID;
            const int64_t G = nchunks * URH_NOISE_SLICES;
            for (int64_t g0 = 0; g0 < G;) {
                int64_t a, b, s0, s1;
                noise_slice(n, ccs, nchunks, g0, &a, &b);
                int64_t g1 = g0 + 1;
                for (; g1 < G; g1++) {
                    noise_slice(n, ccs, nchunks, g1, &s0, &s1);
                    if (s1 - a > cs) break;
                    b = s1;
                }
                out.push_back({g0, g1, a, b});
                g0 = g1;
            }
            return URH_OK;
        }
        case URH_FILTER_STFT:
        case URH_FILTER_DB: {   // frame f reads x[f hop .. f hop + W - 1]
            const int64_t W = p0, hop = p1;
            if (W <= 0 || hop <= 0) return URH_ERR_INVALID;
            const int64_t fpc = frames_per_chunk(cs, hop);
            for (int64_t f0 = 0; f0 < out_len; f0 += fpc) {
                const int64_t f1 = f0 + fpc < out_len ? f0 + fpc : out_len;
                const int64_t b = clamp64((f1 - 1) * hop + W, 0, n);
                out.push_back({f0, f1, clamp64(f0 * hop, 0, b), b});
            }
            return URH_OK;
        }
        case URH_FILTER_IMAGES: {
            // Outputs are the frames of all segments in segment order (the images back to back).  Whole segments are grouped while
            // the group's samples fit a chunk and its frames fit frames_per_chunk; a segment that fits neither alone is cut by frames
            // into pieces of frames_per_chunk frames (what urh_spectrogram_db does with a window of frames).  A chunk within one
            // segment (a piece, or a group of one) uploads exactly the samples its frames read, which may end before the segment does.
            const int64_t W = p0, hop = p1;
            if (W <= 0 || hop <= 0 || nseg < 0 || (nseg > 0 && (!h_seg_start || !h_seg_len))) return URH_ERR_INVALID;
            const int64_t fpc = frames_per_chunk(cs, hop);
            auto reach = [&](int64_t f1, int64_t len) { return (f1 - 1) * hop + W < len ? (f1 - 1) * hop + W : len; };   // read by frames < f1
            int64_t k = 0;              // frames before segment s
            int64_t g0 = -1, ga = 0, gb = 0;   // the open group: its first frame and its sample window
            int gn = 0;                        // its segments
            auto close = [&]() {
                if (g0 >= 0) {
                    if (gn == 1) gb = ga + reach(k - g0, gb - ga);
                    out.push_back({g0, k, ga, gb});
                }
                g0 = -1;
                gn = 0;
            };
            for (int s = 0; s < nseg; s++) {
                const int64_t st = h_seg_start[s], len = h_seg_len[s];
                if (st < 0 || len < 0 || st + len > n) return URH_ERR_INVALID;
                const int64_t F = frames_of(len, W, hop);
                if (len > cs || F > fpc) {
                    close();
                    for (int64_t f0 = 0; f0 < F; f0 += fpc) {
                        const int64_t f1 = f0 + fpc < F ? f0 + fpc : F;
                        out.push_back({k + f0, k + f1, st + f0 * hop, st + reach(f1, len)});
                    }
                    k += F;
                    continue;
                }
                if (g0 >= 0) {
                    const int64_t a = ga < st ? ga : st, b = gb > st + len ? gb : st + len;
                    if (b - a > cs || k + F - g0 > fpc) close();
                }
                if (g0 < 0) {
                    g0 = k; ga = st; gb = st + len;
                } else {
                    ga = ga < st ? ga : st;
                    gb = gb > st + len ? gb : st + len;
                }
                gn++;
                k += F;
            }
            close();
            return URH_OK;
        }
        default: return URH_ERR_INVALID;
    }
}

extern "C" int urh_stream_windows(int entry, int64_t n, int64_t out_len, int64_t p0, int64_t p1, int64_t chunk_samples,
                                  const int64_t* h_seg_start, const int64_t* h_seg_len, int nseg, int64_t* h_win, int64_t cap, int64_t* count) {
    if (!count) return URH_ERR_INVALID;
    std::vector<UrhWindow> w;
    URH_CHECK(urh_filter_windows(entry, n, out_len, p0, p1, chunk_samples, h_seg_start, h_seg_len, nseg, w));
    *count = (int64_t)w.size();
    if (!h_win) return URH_OK;
    if ((int64_t)w.size() > cap) return URH_ERR_INVALID;
    memcpy(h_win, w.data(), w.size() * sizeof(UrhWindow));
    return URH_OK;
}

// The op order of a streamed call, 7 int64 per op {kind, chunk, slot, k0, k1, a, b}.  Op semantics (stream_run and the host model of
// tests/test_stream_filter_plan_cpu.py):
//   upload(c, s)   copy stream 0: waits for the last compute recorded on slot s, copies, records "uploaded" on s
//   compute(c, s)  compute stream: waits for "uploaded" on s (uploading calls) and for the last download recorded on s (calls whose
//                  downloads read the slot), runs the chunk, records "computed" on s
//   download(c, s) copy stream 1: waits for "computed" on s, copies the chunk's outputs out, records "downloaded" on s
// Uploads run R - 1 chunks ahead: the upload of chunk c + R - 1 is issued before compute(c), into the slot compute(c - 1) released.
extern "C" int urh_stream_window_schedule(const int64_t* h_win, int64_t chunks, int ring, int flags, int64_t* h_ops, int64_t cap,
                                          int64_t* count) {
    if (!count || chunks < 0 || (chunks > 0 && !h_win) || ring < 2 || ring > URH_STREAM_MAX_RING) return URH_ERR_INVALID;
    const bool up = flags & URH_STREAM_UPLOAD, down = flags & URH_STREAM_DOWNLOAD;
    int64_t k = 0;
    auto emit = [&](int64_t kind, int64_t c) {
        if (h_ops && k < cap) {
            int64_t* o = h_ops + 7 * k;
            o[0] = kind; o[1] = c; o[2] = c % ring;
            memcpy(o + 3, h_win + 4 * c, 4 * sizeof(int64_t));
        }
        k++;
    };
    if (up)
        for (int64_t c = 0; c < ring - 1 && c < chunks; c++) emit(URH_OP_UPLOAD, c);
    for (int64_t c = 0; c < chunks; c++) {
        if (up && c + ring - 1 < chunks) emit(URH_OP_UPLOAD, c + ring - 1);
        emit(URH_OP_COMPUTE, c);
        if (down) emit(URH_OP_DOWNLOAD, c);
    }
    *count = k;
    return (h_ops && k > cap) ? URH_ERR_INVALID : URH_OK;
}

// ---- device bytes --------------------------------------------------------------------------------------------------------------------
// scratch of a window call of nf frames (spectrogram.cu stft_run): the fused kernel's twiddles, or the cuFFT path's batch of complex128
// frames (at most 512 MiB) and a work area of the same size for cuFFT
static int64_t frames_work(int64_t W, int64_t nf) {
    const int64_t max_batch = ((int64_t)512 << 20) / (W * 16) > 0 ? ((int64_t)512 << 20) / (W * 16) : 1;
    const int64_t batch = nf < max_batch ? (nf > 0 ? nf : 1) : max_batch;
    return r256(W * 16) + 2 * r256(batch * W * 16);
}
// the composed image path's dB rows (urh_spectrogram_bgra: at most 256 MiB) and the fused path's segment table
static int64_t image_work(int64_t W, int64_t nf) {
    const int64_t rows = ((int64_t)256 << 20) / (W * 4) > 0 ? ((int64_t)256 << 20) / (W * 4) : 1;
    return r256((nf < rows ? nf : rows) * W * 4) + r256(nf * 40);
}

static int out_bytes_dc(int dtype) { return dtype == URH_DT_F32 ? 8 : 16; }

FilterStreamSizes urh_filter_stream_sizes(int entry, int64_t n, int64_t out_len, int dtype, int64_t p0, int64_t p1, int64_t p2,
                                          int64_t chunk_samples) {
    (void)out_len;
    FilterStreamSizes z{0, 0, 0, 0};
    int64_t cs = filter_chunk(chunk_samples);
    switch (entry) {
        case URH_FILTER_CONVOLVE:
            z.in_slot = r256((cs + p0 - 1) * 8);
            z.out_slot = r256(cs * 8);
            z.extra = r256(p0 * 16);
            break;
        case URH_FILTER_FIR: {
            const int64_t h = p0 > 1 ? p0 - 1 : 0;
            if (cs < h) cs = h;
            z.in_slot = r256((cs + h) * 8);
            z.out_slot = r256(cs * 8);
            z.extra = r256((p0 > 1 ? p0 : 1) * 8);
            break;
        }
        case URH_FILTER_DC:
            z.in_slot = r256(cs * urh_iq_bytes(dtype));
            z.out_slot = r256(cs * out_bytes_dc(dtype));
            z.work = 3 * r256(4096 * 16);   // column partials of up to 4096 blocks, the sums, the mean
            break;
        case URH_FILTER_NOISE:   // the slot of the largest window; the slices' partials and the chunks' sums and maxima
            z.in_slot = r256(noise_slot_samples(p0, p1, chunk_samples) * urh_iq_bytes(dtype));
            z.out_slot = 0;
            z.extra = 2 * r256(p1 * URH_NOISE_SLICES * 8) + 2 * r256(p1 * 8);
            break;
        case URH_FILTER_CONVERT:
            z.in_slot = r256(cs * urh_iq_bytes(dtype));
            z.out_slot = r256(cs * urh_iq_bytes((int)p0));
            break;
        case URH_FILTER_STFT:
        case URH_FILTER_DB: {
            const int64_t fpc = frames_per_chunk(cs, p1);
            const int64_t in = (fpc - 1) * p1 + p0;
            z.in_slot = r256((in < n ? in : n) * 8);
            z.out_slot = r256(fpc * p0 * (entry == URH_FILTER_STFT ? 16 : 4));
            z.extra = r256(p0 * 8);
            z.work = frames_work(p0, fpc);
            break;
        }
        case URH_FILTER_IMAGES: {
            const int64_t fpc = frames_per_chunk(cs, p1);
            const int64_t in = (fpc - 1) * p1 + p0 > cs ? (fpc - 1) * p1 + p0 : cs;
            z.in_slot = r256((in < n ? in : n) * 8);
            z.out_slot = r256(fpc * p0 * 4);
            z.extra = r256(p0 * 8) + r256(p2 * 4);   // the window and the colormap (p2 BGRA entries)
            z.work = frames_work(p0, fpc) + image_work(p0, fpc);
            break;
        }
        default: break;
    }
    return z;
}

static bool filter_args_ok(int entry, int64_t n, int64_t out_len, int dtype, int64_t p0, int64_t p1, int64_t p2) {
    if (n < 0 || out_len < 0) return false;
    switch (entry) {
        case URH_FILTER_CONVOLVE: return p0 >= 1 && p1 >= 0;
        case URH_FILTER_FIR: return p0 >= 0;
        case URH_FILTER_DC: return urh_iq_bytes(dtype) != 0;
        case URH_FILTER_NOISE: return urh_iq_bytes(dtype) != 0 && p0 >= 1 && p1 >= 1 && p0 * p1 <= n;
        case URH_FILTER_CONVERT: return urh_iq_bytes(dtype) != 0 && urh_iq_bytes((int)p0) != 0;
        case URH_FILTER_STFT:
        case URH_FILTER_DB: return p0 > 0 && p1 > 0;
        case URH_FILTER_IMAGES: return p0 > 0 && p1 > 0 && p2 > 0;
        default: return false;
    }
}

// resident: what the resident entry needs for a host capture (the capture, the whole output, the scratch of one call over all of it)
extern "C" int urh_stream_filter_footprint(int entry, int64_t n, int64_t out_len, int dtype, int64_t p0, int64_t p1, int64_t p2,
                                           int64_t chunk_samples, int ring, int resident, int64_t* bytes) {
    if (!bytes || !filter_args_ok(entry, n, out_len, dtype, p0, p1, p2)) return URH_ERR_INVALID;
    if (!resident && (ring < 2 || ring > URH_STREAM_MAX_RING)) return URH_ERR_INVALID;
    if (resident) {
        int64_t b = URH_ARENA_BLOCK;
        switch (entry) {
            case URH_FILTER_CONVOLVE: b += r256(n * 8) + r256(out_len * 8) + r256(p0 * 16); break;
            case URH_FILTER_FIR: b += 2 * r256(n * 8) + r256((p0 > 1 ? p0 : 1) * 8); break;
            case URH_FILTER_DC: b += r256(n * urh_iq_bytes(dtype)) + r256(n * out_bytes_dc(dtype)) + 3 * r256(4096 * 16); break;
            // the capture uploaded whole, the partials and results in the arena (urh_noise_chunk_stats_iq)
            case URH_FILTER_NOISE: b += r256(n * urh_iq_bytes(dtype)) + 2 * r256(p1 * URH_NOISE_SLICES * 8) + 2 * r256(p1 * 8); break;
            case URH_FILTER_CONVERT: b += r256(n * urh_iq_bytes(dtype)) + r256(n * urh_iq_bytes((int)p0)); break;
            case URH_FILTER_STFT:
            case URH_FILTER_DB:
                b += r256(n * 8) + r256(out_len * p0 * (entry == URH_FILTER_STFT ? 16 : 4)) + r256(p0 * 8) + frames_work(p0, out_len);
                break;
            case URH_FILTER_IMAGES:
                b += r256(n * 8) + r256(out_len * p0 * 4) + r256(p0 * 8) + r256(p2 * 4) + frames_work(p0, out_len) +
                     image_work(p0, out_len);
                break;
        }
        *bytes = b;
        return URH_OK;
    }
    const FilterStreamSizes z = urh_filter_stream_sizes(entry, n, out_len, dtype, p0, p1, p2, chunk_samples);
    *bytes = ring * (z.in_slot + z.out_slot) + z.extra + stream_arena_bytes(z.work);
    return URH_OK;
}

int urh_filter_stream_check(urh_ctx* ctx, int64_t n, int ring) {
    if (n < 0) URH_FAIL(ctx, URH_ERR_INVALID, "streamed filter: negative length");
    if (ring < 2 || ring > URH_STREAM_MAX_RING) URH_FAIL(ctx, URH_ERR_INVALID, "streamed filter: ring of %d slots (2 .. 8)", ring);
    return URH_OK;
}
