// Pulse table -> bit arrays on the GPU (SURVEY §8f row 1): ProtocolAnalyzer._ppseq_to_bits (ProtocolAnalyzer.py:323-414).
//
// The reference walks the (kind, num_samples) rows in a Python loop.  Restated as array operations:
//   num_symbols = int(ns / sps) (+1 if the fraction exceeds 0.5)                                        (:349-353)
//   row types:  D data row (kind >= 0): emits number_to_bits(kind) * num_symbols                         (:392-404)
//               Z short pause (kind == -1, num_symbols <= pause_threshold or pause_threshold == 0): zeros (:356-364)
//               L long pause: closes the running message if it has seen data, else drops the collected bits (:366-390)
//   => L rows cut the table into segments; a segment is a message iff it holds a D row with num_symbols > 0; its bits are
//      everything its rows emit; pause = the closing L row's length; bit_sample_pos = start of every bit plus
//      (total, total + ns) of the closing row, or (total) for the message that ends the table                 (:377-381, :406-412)
//   a table that starts with a pause skips that row but keeps its length in `total`                          (:335-339)
// Every step is a map or a prefix sum over rows; the bits are then expanded with one thread per output bit.
#include "common.cuh"
#include "tilescan.cuh"

enum { PP_SKIP = 0, PP_DATA = 1, PP_ZERO = 2, PP_LONG = 3 };

__global__ void k_pp_rows(const int64_t* __restrict__ rows, int64_t k, double sps, int bps, int pause_threshold,
                          int64_t* __restrict__ ns_out, int64_t* __restrict__ nbits, int64_t* __restrict__ sep,
                          uint8_t* __restrict__ type, uint8_t* __restrict__ has_data) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const int64_t kind = rows[2 * i], ns = rows[2 * i + 1];
    const int64_t first = (rows[0] == -1) ? 1 : 0;
    ns_out[i] = ns;
    int t = PP_SKIP;
    int64_t nb = 0;
    uint8_t hd = 0;
    if (i >= first) {
        // Python: num_symbols_float = num_samples / samples_per_symbol (true division, double)
        const double f = (double)ns / sps;
        int64_t nsym = (int64_t)f;
        if (f - (double)nsym > 0.5) nsym++;
        if (kind == -1) {
            if (nsym <= pause_threshold || pause_threshold == 0) { t = PP_ZERO; nb = nsym * bps; }
            else t = PP_LONG;
        } else {
            t = PP_DATA;
            nb = nsym * bps;
            hd = nsym > 0 ? 1 : 0;
        }
    }
    nbits[i] = nb;
    sep[i] = (t == PP_LONG) ? 1 : 0;
    type[i] = (uint8_t)t;
    has_data[i] = hd;
}

__global__ void k_pp_mark(const int64_t* __restrict__ seg, const uint8_t* __restrict__ has_data, int64_t k, int64_t* __restrict__ seg_has) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k && has_data[i]) seg_has[seg[i]] = 1;
}

// scan elements: in[i]; out[i] = exclusive prefix (in == out: in place)
struct PpPrefix {
    const int64_t* in;
    int64_t* out;
    __device__ __forceinline__ int64_t load(int64_t i) const { return in[i]; }
    __device__ __forceinline__ void post(int64_t i, const int64_t& excl, const int64_t&) const { out[i] = excl; }
};
// a row's bits count only if its segment is a message; nbits[i] becomes the row's bit offset
struct PpBitOffsets {
    const int64_t* seg;
    const int64_t* seg_has;
    int64_t* nbits;
    __device__ __forceinline__ int64_t load(int64_t i) const { return seg_has[seg[i]] ? nbits[i] : 0; }
    __device__ __forceinline__ void post(int64_t i, const int64_t& excl, const int64_t&) const { nbits[i] = excl; }
};
// 8 items per thread: on a table of 10^7 rows that runs each scan about a fifth faster than 16 (H100)
static int pp_scan(urh_ctx* ctx, const int64_t* in, int64_t* out, int64_t k, int64_t* d_total) {
    PpPrefix f;
    f.in = in; f.out = out;
    return urhts::scan<int64_t, urhts::AddI64, PpPrefix, 8>(ctx, k, (int64_t)0, urhts::AddI64(), f, d_total);
}

// mailbox: {n_msgs, total_bits, final_open, n_long}
__global__ void k_pp_counts(const int64_t* __restrict__ seg_has, const int64_t* __restrict__ d_nlong, const int64_t* __restrict__ d_nmsg,
                            const int64_t* __restrict__ d_bits, int64_t* __restrict__ out) {
    out[0] = *d_nmsg;
    out[1] = *d_bits;
    out[2] = seg_has[*d_nlong];
    out[3] = *d_nlong;
}

__global__ void k_pp_meta(const int64_t* __restrict__ rows, const uint8_t* __restrict__ type, const int64_t* __restrict__ seg,
                          const int64_t* __restrict__ seg_has, const int64_t* __restrict__ seg_msg, const int64_t* __restrict__ bitoff,
                          const int64_t* __restrict__ total, int64_t k, int64_t n_msgs, int64_t total_bits, int final_open,
                          int64_t total_end, int write_pos, int64_t* __restrict__ msg_off, int64_t* __restrict__ pauses,
                          int64_t* __restrict__ pos) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        msg_off[0] = 0;
        if (final_open) {
            const int64_t m = n_msgs - 1;
            msg_off[n_msgs] = total_bits;
            pauses[m] = (rows[2 * (k - 1)] == -1) ? rows[2 * (k - 1) + 1] : 0;
            if (write_pos) pos[total_bits + 2 * m] = total_end;
        }
    }
    if (i >= k || type[i] != PP_LONG) return;
    const int64_t s = seg[i];
    if (!seg_has[s]) return;
    const int64_t m = seg_msg[s];
    const int64_t ns = rows[2 * i + 1];
    msg_off[m + 1] = bitoff[i];
    pauses[m] = ns;
    if (write_pos) {
        pos[bitoff[i] + 2 * m] = total[i];
        pos[bitoff[i] + 2 * m + 1] = total[i] + ns;
    }
}

__global__ void k_pp_expand(const int64_t* __restrict__ rows, const uint8_t* __restrict__ type, const int64_t* __restrict__ seg,
                            const int64_t* __restrict__ seg_msg, const int64_t* __restrict__ bitoff, const int64_t* __restrict__ total,
                            int64_t k, int64_t total_bits, int bps, int64_t samples_per_bit, int write_pos,
                            uint8_t* __restrict__ bits, int64_t* __restrict__ pos) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total_bits) return;
    // last row whose bit offset is <= g (rows that emit nothing share their successor's offset)
    int64_t lo = 0, hi = k;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (bitoff[mid] <= g) lo = mid; else hi = mid;
    }
    const int64_t i = lo;
    const int64_t b = g - bitoff[i];
    uint8_t v = 0;
    if (type[i] == PP_DATA) {
        const int64_t kind = rows[2 * i];
        v = (uint8_t)((kind >> (bps - 1 - (int)(b % bps))) & 1);   // number_to_bits: MSB first, bps digits
    }
    bits[g] = v;
    if (write_pos) pos[g + 2 * seg_msg[seg[i]]] = total[i] + b * samples_per_bit;
}

// d_rows: int64[k,2] pulse table on the device (NULL: the table the last digitizer call left in the context).
// Results stay in the context's scratch arena until the next call; urh_fetch_bits copies them out.
// *n_pos = length of the flat bit_sample_pos array (0 when write_pos == 0).
extern "C" int urh_ppseq_to_bits(urh_ctx* ctx, const int64_t* d_rows, int64_t k, uint32_t samples_per_symbol, uint8_t bits_per_symbol,
                                 int pause_threshold, int write_pos, int64_t* n_msgs, int64_t* n_bits, int64_t* n_pos) {
    if (!n_msgs || !n_bits || !n_pos) return URH_ERR_INVALID;
    *n_msgs = 0; *n_bits = 0; *n_pos = 0;
    if (!d_rows) {
        d_rows = ctx->pulses;
        if (k > ctx->pulses_k) URH_FAIL(ctx, URH_ERR_INVALID, "the context holds %lld pulse rows, %lld requested", (long long)ctx->pulses_k, (long long)k);
    }
    if (samples_per_symbol == 0 || bits_per_symbol == 0 || bits_per_symbol > 8) URH_FAIL(ctx, URH_ERR_INVALID, "samples_per_symbol > 0 and 1 <= bits_per_symbol <= 8 required");
    urh_arena_reset(ctx);
    ctx->bits_valid = 0;
    if (k <= 0) {
        ctx->bits_valid = 1; ctx->bits_nmsg = 0; ctx->bits_total = 0; ctx->bits_npos = 0;
        return URH_OK;
    }
    int64_t *total, *nbits, *seg, *seg_has, *seg_msg, *d_cnt, *mail;
    uint8_t *type, *has_data;
    URH_CHECK(urh_arena(ctx, (size_t)k, &total));
    URH_CHECK(urh_arena(ctx, (size_t)k, &nbits));
    URH_CHECK(urh_arena(ctx, (size_t)k, &seg));
    URH_CHECK(urh_arena(ctx, (size_t)k + 2, &seg_has));
    URH_CHECK(urh_arena(ctx, (size_t)k + 2, &seg_msg));
    URH_CHECK(urh_arena(ctx, 8, &d_cnt));   // [0] total samples, [1] long pauses, [2] messages, [3] bits
    URH_CHECK(urh_arena(ctx, 8, &mail));
    URH_CHECK(urh_arena(ctx, (size_t)k, &type));
    URH_CHECK(urh_arena(ctx, (size_t)k, &has_data));
    const unsigned g = (unsigned)urh_div_up(k, 256);
    URH_LAUNCH(ctx, k_pp_rows, g, 256, 0, d_rows, k, (double)samples_per_symbol, (int)bits_per_symbol, pause_threshold, total, nbits, seg, type, has_data);
    URH_CHECK(pp_scan(ctx, total, total, k, d_cnt + 0));
    URH_CHECK(pp_scan(ctx, seg, seg, k, d_cnt + 1));
    URH_CUDA(ctx, cudaMemsetAsync(seg_has, 0, ((size_t)k + 2) * sizeof(int64_t), ctx->stream));
    URH_LAUNCH(ctx, k_pp_mark, g, 256, 0, seg, has_data, k, seg_has);
    URH_CHECK(pp_scan(ctx, seg_has, seg_msg, k + 1, d_cnt + 2));
    PpBitOffsets fb;
    fb.seg = seg; fb.seg_has = seg_has; fb.nbits = nbits;
    URH_CHECK((urhts::scan<int64_t, urhts::AddI64, PpBitOffsets, 8>(ctx, k, (int64_t)0, urhts::AddI64(), fb, d_cnt + 3)));
    URH_LAUNCH(ctx, k_pp_counts, 1, 1, 0, seg_has, d_cnt + 1, d_cnt + 2, d_cnt + 3, mail);
    int64_t h[4], total_end = 0;
    URH_CHECK(urh_read_i64(ctx, mail, 4, h));
    URH_CHECK(urh_read_i64(ctx, d_cnt, 1, &total_end));
    const int64_t M = h[0], B = h[1];
    const int final_open = h[2] ? 1 : 0;
    const int64_t P = write_pos ? (B + 2 * M - (final_open ? 1 : 0)) : 0;
    uint8_t* bits;
    int64_t *msg_off, *pauses, *pos;
    URH_CHECK(urh_arena(ctx, (size_t)B + 16, &bits));
    URH_CHECK(urh_arena(ctx, (size_t)M + 2, &msg_off));
    URH_CHECK(urh_arena(ctx, (size_t)M + 2, &pauses));
    URH_CHECK(urh_arena(ctx, (size_t)P + 4, &pos));
    if (M > 0) {
        URH_LAUNCH(ctx, k_pp_meta, g, 256, 0, d_rows, type, seg, seg_has, seg_msg, nbits, total, k, M, B, final_open, total_end, write_pos,
                   msg_off, pauses, pos);
        if (B > 0)
            URH_LAUNCH(ctx, k_pp_expand, (unsigned)urh_div_up(B, 256), 256, 0, d_rows, type, seg, seg_msg, nbits, total, k, B, (int)bits_per_symbol,
                       (int64_t)((int)(samples_per_symbol / bits_per_symbol)), write_pos, bits, pos);
    }
    ctx->bits_valid = 1;
    ctx->bits_nmsg = M; ctx->bits_total = B; ctx->bits_npos = P;
    ctx->bits_ptr = bits; ctx->bits_msg_off = msg_off; ctx->bits_pauses = pauses; ctx->bits_pos = pos;
    *n_msgs = M; *n_bits = B; *n_pos = P;
    return URH_OK;
}

// h_bits: uint8[n_bits]; h_msg_off: int64[n_msgs + 1] (message m = bits[off[m]:off[m+1]], its positions
// pos[off[m] + 2m : off[m+1] + 2m + 2], one entry fewer for a last message that is not closed by a pause row);
// h_pauses: int64[n_msgs]; h_pos: int64[n_pos] or NULL.
extern "C" int urh_fetch_bits(urh_ctx* ctx, uint8_t* h_bits, int64_t* h_msg_off, int64_t* h_pauses, int64_t* h_pos) {
    if (!ctx->bits_valid) URH_FAIL(ctx, URH_ERR_INVALID, "urh_ppseq_to_bits must precede urh_fetch_bits");
    const int64_t M = ctx->bits_nmsg, B = ctx->bits_total, P = ctx->bits_npos;
    if (M == 0) {
        if (h_msg_off) h_msg_off[0] = 0;
        return URH_OK;
    }
    if (h_bits && B) URH_CUDA(ctx, cudaMemcpyAsync(h_bits, ctx->bits_ptr, (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
    if (h_msg_off) URH_CUDA(ctx, cudaMemcpyAsync(h_msg_off, ctx->bits_msg_off, (size_t)(M + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (h_pauses) URH_CUDA(ctx, cudaMemcpyAsync(h_pauses, ctx->bits_pauses, (size_t)M * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (h_pos && P) URH_CUDA(ctx, cudaMemcpyAsync(h_pos, ctx->bits_pos, (size_t)P * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}

extern "C" const uint8_t* urh_bits_device_ptr(urh_ctx* ctx) { return ctx->bits_valid ? (const uint8_t*)ctx->bits_ptr : nullptr; }
