// Spectrogram: STFT -> fftshift -> dB (reference: Spectrogram.stft Spectrogram.py:94-116,
// __calculate_spectrogram :156-162, util.arr2decibel util.pyx:38-48).
//
// The reference multiplies complex frames by np.hanning in float64 and runs numpy's complex128 FFT, then casts
// to complex64 and takes 10*log10f(|X|^2) in float32.  To keep the weak bins (down to ~-100 dB below the peak)
// within the stated 1e-3 dB, the FFT is done in double.  Power-of-two windows of 128 .. 4096 points (URH's: 1024) take ONE fused
// kernel (window -> shared-memory FFT -> scale / fftshift / cast / dB / flip, see k_stft_r16); other sizes use cuFFT Z2Z — for the
// FFT only, as the north_star prescribes — between two hand-written kernels, in batches that bound the working set.
#include "common.cuh"
#include "stream_ring.cuh"

#include <cufft.h>
#include <limits.h>
#include <math.h>

#include <algorithm>

#define URH_CUFFT(ctx, call)                                                                    \
    do {                                                                                        \
        cufftResult r__ = (call);                                                               \
        if (r__ != CUFFT_SUCCESS) {                                                             \
            snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d: %s -> cufft error %d", __FILE__, __LINE__, #call, (int)r__); \
            return URH_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

// sample * window value as the STFT's input.  A non-finite sample gives NaN + NaN j, so every bin of each frame that reads it is
// NaN + NaN j whatever the order of the butterflies, as in the reference: numpy promotes the window to complex, so (inf, 0) * g is
// (inf, NaN) and inf * 0 is NaN, and its transform of the frames spreads that to both parts of every bin (DESIGN.md §4.6).  A real
// product would leave finite and infinite bins: +inf dB where the reference has NaN.
__device__ __forceinline__ double2 stft_windowed(float2 s, double g) {
    if (!(isfinite(s.x) && isfinite(s.y))) return make_double2(__longlong_as_double(0x7ff8000000000000ll), __longlong_as_double(0x7ff8000000000000ll));
    return make_double2((double)s.x * g, (double)s.y * g);
}

// frames[f][w] = x[(f0+f)*hop + w] * window[w]  (complex128; samples beyond n are zero: Spectrogram.py:102-103)
__global__ void k_stft_window(const float2* __restrict__ x, int64_t n, int W, int hop, const double* __restrict__ window,
                              int64_t f0, int64_t nframes, double2* __restrict__ frames) {
    const int64_t total = nframes * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int64_t f = idx / W;
        const int w = (int)(idx - f * W);
        const int64_t i = (f0 + f) * hop + w;
        double2 v = make_double2(0.0, 0.0);
        if (i < n) v = stft_windowed(x[i], window[w]);
        frames[idx] = v;
    }
}

// out[f][w] = X[f][w] / W   (Spectrogram.stft result, complex128)
__global__ void k_stft_scale(const double2* __restrict__ X, int W, int64_t total, double2* __restrict__ out) {
    const double inv = (double)W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const double2 v = X[idx];
        out[idx] = make_double2(v.x / inv, v.y / inv);
    }
}

// out[f][j] = dB(shifted[f][W-1-j]), shifted[j] = X[(j + W - W/2... np.fft.fftshift: shifted[j] = X[(j - W/2) mod W] for even/odd W
__global__ void k_stft_db(const double2* __restrict__ X, int W, int64_t nframes, float* __restrict__ out) {
    const int64_t total = nframes * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const double dW = (double)W;
    const int half = W / 2;  // fftshift moves index n//2.. to the front: shifted[j] = X[(j + (W+1)/2) % W]
    const int shift = (W + 1) / 2;
    (void)half;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int64_t f = idx / W;
        const int j = (int)(idx - f * W);
        const int js = W - 1 - j;                 // fliplr
        const int src = (js + shift) % W;         // fftshift
        const double2 v = X[f * W + src];
        const float re = (float)(v.x / dW), im = (float)(v.y / dW);   // complex128 / W, then astype(complex64)
        out[idx] = __fmul_rn(10.0f, log10f(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im))));
    }
}

// ---- fused path (power-of-two windows): window -> FFT in shared memory -> scale / fftshift / dB, W / 16 threads per frame ------
// The cuFFT path above moves every frame through HBM three times as complex128 (window kernel -> Z2Z -> dB kernel: 36 GB for
// 2^28 samples at W = 1024, hop = 512).  Here a frame is read once as complex64 (the 50 % overlap with its neighbour comes from
// L2), transformed in double in shared memory (Stockham autosort, radix-16 passes + one radix-2 / 4 / 8 pass, see k_stft_r16)
// and written once as float32 dB (or complex128 for urh_stft): 8 + 8 B/sample at the reference's parameters.
// tw[q] = exp(-2 pi i q / W), q < W, built once per window size with sincospi (double).
__global__ void k_fft_twiddles(int W, double2* __restrict__ tw) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= W) return;
    double s, c;
    sincospi(-2.0 * (double)q / (double)W, &s, &c);
    tw[q] = make_double2(c, s);
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}

// ---- MODE 2: the spectrogram image (Spectrogram.create_spectrogram_image / create_image_segments, Spectrogram.py:164-190) -----
// Each bin takes the dB map's steps (scale, fftshift, complex64 cast, 10 log10f, fliplr), then k_bgra_lookup's (bgra_index), and
// only the 4-byte colormap entry is written.  One launch covers every frame of every segment of a capture: seg[5 s ..] =
// {first sample, end sample, frames, first block, first pixel} of segment s; no frame reads at or past its segment's end (the
// zero-padding of Spectrogram.py:102-103 per segment).  A block owns STFT_IMG_FPB consecutive frames of one segment.
//   transpose = 0: image [W][F] (row r = dB column r, column f = frame f).  The block keeps its frames' colormap indices in shared
//                  memory ([W][FPB] uint16) and writes each row's FPB pixels together: 8 frames = 32-byte row segments.  uint16
//                  rather than the 4-byte entries keeps W = 4096 in shared memory: 139 KB (radix-16 FFT buffers) + 64 KB indices
//                  + 4 KB colormap = 204 KB of the 227 KB a block may have; 4-byte entries would need 267 KB.  Colormaps of more
//                  than 65536 entries therefore take the composed path (urh_spectrogram_bgra).
//   transpose = 1: image [F][W] (np.flipud(dB.T) before the look-up: bins in fftshift order); each frame's row is written as it is
//                  computed, coalesced.
// padded shared-memory index of the radix-16 kernel (one element every 16; see k_stft_r16)
__device__ __forceinline__ int stft_pad(int i) { return i + (i >> 4); }
// k_stft_r16 runs W / 16 threads per frame; its blocks hold several frames where that is less than a warp (W = 128, 256)
constexpr int stft_frames(int W) { return W / 16 >= 32 ? 1 : 32 / (W / 16); }
// the thread's frame within its block, and its lane among that frame's W / 16 threads
template <int W>
__device__ __forceinline__ int stft_group() { return stft_frames(W) > 1 ? (int)(threadIdx.x / (W / 16)) : 0; }
template <int W>
__device__ __forceinline__ int stft_lane() { return stft_frames(W) > 1 ? (int)(threadIdx.x % (W / 16)) : (int)threadIdx.x; }
constexpr int STFT_IMG_FPB = 8;
struct StftImage {
    const int64_t* seg;
    int nseg;
    const uint32_t* cmap;
    int entries;
    float data_min, range;
    int transpose;
};

// Spectrogram.apply_bgra_lookup per value: float32 subtract, divide, multiply, truncate toward zero (astype(int)), np.take(mode="clip");
// numpy's cast is exact for |v| < 2^63; NaN, infinities and everything else become INT64_MIN, which mode="clip" maps to entry 0
__device__ __forceinline__ int bgra_index(float v, float data_min, float range, float scale, int L, int normalize) {
    if (normalize) v = __fmul_rn(scale, __fdiv_rn(__fsub_rn(v, data_min), range));
    long long k = (v == v && fabsf(v) < 0x1p63f) ? (long long)v : LLONG_MIN;
    k = k < 0 ? 0 : (k > L - 1 ? L - 1 : k);
    return (int)k;
}

// fft(base, end) runs the FFT of the thread's frame (samples base .. base + W - 1, zeros at and past end) and returns the (padded)
// buffer holding X; `tail` is the shared memory after the FFT buffers
template <int W, typename Fft>
__device__ __forceinline__ void stft_image_block(const StftImage& img, int hop, Fft fft, unsigned char* tail, uint32_t* __restrict__ out) {
    constexpr int FPB = STFT_IMG_FPB;
    constexpr int T = W / 16, G = stft_frames(W), NT = G * T;
    const int64_t blk = blockIdx.x;
    int lo = 0, hi = img.nseg - 1;   // the last segment whose first block is <= blk
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (img.seg[5 * mid + 3] <= blk) lo = mid;
        else hi = mid - 1;
    }
    const int64_t* sg = img.seg + 5 * lo;
    const int64_t start = sg[0], end = sg[1], F = sg[2];
    const int64_t f0 = (blk - sg[3]) * FPB;
    const int nf = (int)min((int64_t)FPB, F - f0);
    uint32_t* o = out + sg[4];
    uint16_t* s_idx = (uint16_t*)tail;                       // [W][FPB]
    uint32_t* s_map = (uint32_t*)(tail + W * FPB * sizeof(uint16_t));
    const bool map_smem = img.entries <= 1024;
    if (map_smem)
        for (int i = threadIdx.x; i < img.entries; i += NT) s_map[i] = img.cmap[i];
    __syncthreads();
    const uint32_t* map = map_smem ? s_map : img.cmap;
    const float scale = (float)(img.entries - 1);
    constexpr int shift = (W + 1) / 2;
    const double inv = 1.0 / (double)W;
    for (int k0 = 0; k0 < nf; k0 += G) {   // G frames at a time, one per group of T threads
        const int k = k0 + stft_group<W>();  // k >= nf (the last block of a segment): transformed, not written
        const double2* a = fft(start + (f0 + k) * hop, end);
        if (G == 1 || k < nf) {
            for (int r = stft_lane<W>(); r < W; r += T) {
                const int j = img.transpose ? W - 1 - r : r;            // dB column (fliplr order)
                const int src = ((W - 1 - j) + shift) & (W - 1);        // fliplr, then fftshift
                const double2 v = a[stft_pad(src)];
                const float re = (float)(v.x * inv), im = (float)(v.y * inv);
                const float db = __fmul_rn(10.0f, log10f(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im))));
                const int idx = bgra_index(db, img.data_min, img.range, scale, img.entries, 1);
                if (img.transpose) o[(f0 + k) * W + r] = map[idx];
                else s_idx[r * FPB + k] = (uint16_t)idx;
            }
        }
        __syncthreads();   // the next frames' loads overwrite the FFT buffers
    }
    if (!img.transpose) {
        for (int t = threadIdx.x; t < W * FPB; t += NT) {
            const int r = t / FPB, k = t % FPB;
            if (k < nf) o[(int64_t)r * F + f0 + k] = map[s_idx[t]];
        }
    }
}

// ---- the FFT (W = 2^LOG2W, 128 .. 4096): LOG2W / 4 radix-16 passes, each two radix-4 levels held in registers, then one closing
// pass of radix 2^(LOG2W mod 4) (radix-8 for 128 and 2048, radix-2 for 512, radix-4 for 1024, none for 256 and 4096), so a frame
// crosses shared memory three times at W = 1024 (16 * 16 * 4).  One thread owns 16 points of every pass; W / 16 threads per frame
// (stft_frames frames per block).
// Both buffers are padded by one element every 16 (stft_pad) so that the stride-16 stores of the first pass do not pile onto the
// same banks.
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 cmul_mi(double2 a) { return make_double2(a.y, -a.x); }   // a * (-i)
// forward DFT of length 4, in place
__device__ __forceinline__ void dft4(double2& x0, double2& x1, double2& x2, double2& x3) {
    const double2 s02 = cadd(x0, x2), d02 = csub(x0, x2), s13 = cadd(x1, x3), d13 = cmul_mi(csub(x1, x3));
    x0 = cadd(s02, s13); x1 = cadd(d02, d13); x2 = csub(s02, s13); x3 = csub(d02, d13);
}
// forward DFT of length 2, in place
__device__ __forceinline__ void dft2(double2& x0, double2& x1) {
    const double2 s = cadd(x0, x1), d = csub(x0, x1);
    x0 = s; x1 = d;
}
// forward DFT of length 8, in place: v[c + 2 m] -> columns (DFT4 over m), twiddle w8^(c r), rows (DFT2 over c); natural order out
__device__ __forceinline__ void dft8(double2 (&v)[8]) {
    const double H = 0.70710678118654752440;
    dft4(v[0], v[2], v[4], v[6]);   // now v[c + 2 r] = u_c[r]
    dft4(v[1], v[3], v[5], v[7]);
    v[1 + 2] = cmul(v[1 + 2], make_double2(H, -H));    // c=1, r=1: w8^1
    v[1 + 4] = cmul_mi(v[1 + 4]);                      // w8^2 = -i
    v[1 + 6] = cmul(v[1 + 6], make_double2(-H, -H));   // w8^3
#pragma unroll
    for (int r = 0; r < 4; r++) dft2(v[2 * r], v[2 * r + 1]);   // v[2 r + s] = y[r + 4 s]
    const double2 y[8] = {v[0], v[2], v[4], v[6], v[1], v[3], v[5], v[7]};
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = y[i];
}
// forward DFT of length 16, in place: v[c + 4 r'] -> columns, twiddle w16^(c r), rows; output y[r + 4 s] (natural order)
__device__ __forceinline__ void dft16(double2 (&v)[16]) {
    const double C1 = 0.92387953251128675613, S1 = 0.38268343236508977173, H = 0.70710678118654752440;
#pragma unroll
    for (int c = 0; c < 4; c++) dft4(v[c], v[c + 4], v[c + 8], v[c + 12]);   // now v[c + 4 r] = u_c[r]
    // u_c[r] *= w16^(c r)
    v[1 + 4] = cmul(v[1 + 4], make_double2(C1, -S1));    // c=1, r=1: w^1
    v[1 + 8] = cmul(v[1 + 8], make_double2(H, -H));      // w^2
    v[1 + 12] = cmul(v[1 + 12], make_double2(S1, -C1));  // w^3
    v[2 + 4] = cmul(v[2 + 4], make_double2(H, -H));      // c=2, r=1: w^2
    v[2 + 8] = cmul_mi(v[2 + 8]);                        // w^4 = -i
    v[2 + 12] = cmul(v[2 + 12], make_double2(-H, -H));   // w^6
    v[3 + 4] = cmul(v[3 + 4], make_double2(S1, -C1));    // c=3, r=1: w^3
    v[3 + 8] = cmul(v[3 + 8], make_double2(-H, -H));     // w^6
    v[3 + 12] = cmul(v[3 + 12], make_double2(-C1, S1));  // w^9
    // rows: y[r + 4 s] = sum_c u_c[r] w4^(c s): DFT4 over c for each r; u_c[r] sits at v[c + 4 r]
#pragma unroll
    for (int r = 0; r < 4; r++) dft4(v[4 * r], v[4 * r + 1], v[4 * r + 2], v[4 * r + 3]);   // v[4 r + s] = y[r + 4 s]
}

// frame at x[base ..], samples at and past n are zeros: window -> radix-16 FFT; returns the (padded) buffer holding X
template <int LOG2W>
__device__ __forceinline__ const double2* stft_r16_fft(const float2* __restrict__ x, int64_t n, int64_t base,
                                                       const double* __restrict__ window, const double2* __restrict__ tw,
                                                       double2* s_buf) {
    constexpr int W = 1 << LOG2W;
    constexpr int T = W / 16;                 // threads per frame
    constexpr int PADW = W + W / 16;
    double2* a = s_buf;
    double2* b = s_buf + PADW;
    const int tid = stft_lane<W>();
    {
        float2 sm[16];
        double g[16];
#pragma unroll
        for (int m = 0; m < 16; m++) {
            const int w = tid + T * m;
            const int64_t i = base + w;
            sm[m] = (i < n) ? x[i] : make_float2(0.0f, 0.0f);
            g[m] = window[w];
        }
#pragma unroll
        for (int m = 0; m < 16; m++) a[stft_pad(tid + T * m)] = stft_windowed(sm[m], g[m]);
    }
    __syncthreads();
    constexpr int NPASS16 = LOG2W / 4;
#pragma unroll
    for (int st = 0; st < NPASS16; st++) {
        const int ns = 1 << (4 * st);
        const int k = tid & (ns - 1);
        const int tstep = W / (16 * ns);
        double2 v[16];
#pragma unroll
        for (int m = 0; m < 16; m++) v[m] = a[stft_pad(tid + T * m)];
        if (ns > 1) {
#pragma unroll
            for (int m = 1; m < 16; m++) v[m] = cmul(v[m], tw[m * k * tstep]);
        }
        dft16(v);   // v[4 r + s] = y[r + 4 s]
        const int o = ((tid - k) << 4) + k;
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int q = 0; q < 4; q++) b[stft_pad(o + ns * (r + 4 * q))] = v[4 * r + q];
        __syncthreads();
        double2* t = a; a = b; b = t;
    }
    constexpr int R = 1 << (LOG2W & 3);   // the closing pass: sub-transforms of length W / R left
    if constexpr (R > 1) {
        constexpr int ns = W / R;
        double2 y[16 / R][R];   // 16 / R butterflies of radix R per thread
#pragma unroll
        for (int r = 0; r < 16 / R; r++) {
            const int j = tid + T * r;   // butterfly index < W / R; k = j (ns = W / R > j)
#pragma unroll
            for (int q = 0; q < R; q++) y[r][q] = a[stft_pad(j + ns * q)];
#pragma unroll
            for (int q = 1; q < R; q++) y[r][q] = cmul(y[r][q], tw[q * j]);
            if constexpr (R == 2) dft2(y[r][0], y[r][1]);
            else if constexpr (R == 4) dft4(y[r][0], y[r][1], y[r][2], y[r][3]);
            else dft8(y[r]);
        }
#pragma unroll
        for (int r = 0; r < 16 / R; r++)
#pragma unroll
            for (int q = 0; q < R; q++) b[stft_pad(tid + T * r + ns * q)] = y[r][q];
        __syncthreads();
        double2* t = a; a = b; b = t;
    }
    return a;
}

// MODE 0: out = complex128 [F][W] = X / W;  MODE 1: out = float32 [F][W] dB map (fftshift + fliplr + complex64 cast + 10 log10f);
// MODE 2: the image (img, see StftImage)
// W = 2^LOG2W is compile-time: every loop below is fully unrolled (a thread's 16 loads are in flight together — the first version,
// with run-time W, was bound by the latency of one load after the other — and the index arithmetic of the passes is shifts and masks).
template <int LOG2W, int MODE>
__global__ void __launch_bounds__(stft_frames(1 << LOG2W) * (1 << LOG2W) / 16) k_stft_r16(const float2* __restrict__ x, int64_t n, int hop,
                                                               const double* __restrict__ window, const double2* __restrict__ tw,
                                                               int64_t nframes, void* __restrict__ out_, StftImage img) {
    constexpr int W = 1 << LOG2W;
    constexpr int T = W / 16;                 // threads per frame
    constexpr int PADW = W + W / 16;
    constexpr int G = stft_frames(W);         // frames per block
    extern __shared__ double2 s_buf[];        // two padded buffers per frame (MODE 2: then the image staging)
    double2* buf = s_buf + stft_group<W>() * 2 * PADW;
    if (MODE == 2) {
        stft_image_block<W>(
            img, hop, [&](int64_t base, int64_t end) { return stft_r16_fft<LOG2W>(x, end, base, window, tw, buf); },
            (unsigned char*)(s_buf + 2 * G * PADW), (uint32_t*)out_);
        return;
    }
    const int tid = stft_lane<W>();
    const int64_t f = (int64_t)blockIdx.x * G + stft_group<W>();
    const double2* a = stft_r16_fft<LOG2W>(x, n, f * hop, window, tw, buf);
    if (G > 1 && f >= nframes) return;        // the last block's spare frames (their samples read as zeros)
    const double inv = 1.0 / (double)W;
    if (MODE == 0) {
        double2* out = (double2*)out_ + f * W;
#pragma unroll
        for (int m = 0; m < 16; m++) {
            const int w = tid + T * m;
            const double2 v = a[stft_pad(w)];
            out[w] = make_double2(v.x * inv, v.y * inv);
        }
    } else {
        float* out = (float*)out_ + f * W;
        constexpr int shift = (W + 1) / 2;
#pragma unroll
        for (int m = 0; m < 16; m++) {
            const int j = tid + T * m;
            const int src = ((W - 1 - j) + shift) & (W - 1);   // fliplr, then fftshift
            const double2 v = a[stft_pad(src)];
            const float re = (float)(v.x * inv), im = (float)(v.y * inv);
            out[j] = __fmul_rn(10.0f, log10f(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im))));
        }
    }
}

// the shared-memory kernel serves power-of-two windows of 128 .. 4096 points (W = 4096: 139 KB of FFT buffers), grids of fewer
// than 2^31 blocks (frames, or image blocks: far beyond any capture that fits the device) and colormaps whose indices fit the
// image mode's uint16 staging; everything else takes cuFFT
static bool stft_smem_serves(int W, int64_t blocks, int entries) {
    return (W & (W - 1)) == 0 && W >= 128 && W <= 4096 && blocks < ((int64_t)1 << 31) && entries <= 65536;
}

template <int LOG2W>
static int stft_r16_launch(urh_ctx* ctx, int mode, const float* d_x, int64_t n, int hop, const double* d_window, const double2* tw,
                           int64_t count, void* d_out, const StftImage& img) {
    constexpr int W = 1 << LOG2W, G = stft_frames(W);
    const auto kernel = mode == 0 ? k_stft_r16<LOG2W, 0> : mode == 1 ? k_stft_r16<LOG2W, 1> : k_stft_r16<LOG2W, 2>;
    size_t smem = (size_t)2 * G * (W + W / 16) * sizeof(double2);
    if (mode == 2) smem += (size_t)W * STFT_IMG_FPB * sizeof(uint16_t) + 1024 * sizeof(uint32_t);
    if (smem > 48 * 1024) URH_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t blocks = mode == 2 ? count : urh_div_up(count, G);
    URH_LAUNCH(ctx, kernel, (unsigned)blocks, G * W / 16, smem, (const float2*)d_x, n, hop, d_window, tw, count, d_out, img);
    return URH_OK;
}

// one launch of k_stft_r16 for a window stft_smem_serves: `count` frames (modes 0, 1) or image blocks (mode 2)
static int stft_r16(urh_ctx* ctx, int mode, int W, const float* d_x, int64_t n, int hop, const double* d_window, const double2* tw,
                    int64_t count, void* d_out, const StftImage& img) {
    int log2w = 0;
    while ((1 << log2w) < W) log2w++;
    switch (log2w) {
        case 7: return stft_r16_launch<7>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        case 8: return stft_r16_launch<8>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        case 9: return stft_r16_launch<9>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        case 10: return stft_r16_launch<10>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        case 11: return stft_r16_launch<11>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        case 12: return stft_r16_launch<12>(ctx, mode, d_x, n, hop, d_window, tw, count, d_out, img);
        default: URH_FAIL(ctx, URH_ERR_INVALID, "stft: unsupported window size %d", W);
    }
}

static int ensure_plan(urh_ctx* ctx, int W, int64_t batch) {
    if (ctx->fft_valid && ctx->fft_nfft == W && ctx->fft_batch == batch) return URH_OK;
    if (ctx->fft_valid) {
        cufftDestroy((cufftHandle)ctx->fft_plan);
        ctx->fft_valid = false;
    }
    cufftHandle plan;
    int nfft[1] = {W};
    URH_CUFFT(ctx, cufftPlanMany(&plan, 1, nfft, nullptr, 1, W, nullptr, 1, W, CUFFT_Z2Z, (int)batch));
    URH_CUFFT(ctx, cufftSetStream(plan, ctx->stream));
    ctx->fft_plan = (int)plan;
    ctx->fft_nfft = W;
    ctx->fft_batch = batch;
    ctx->fft_valid = true;
    return URH_OK;
}

// mode 0: d_out = complex128 [F][W] stft (Spectrogram.stft);  mode 1: d_out = float32 [F][W] dB map
static int stft_run(urh_ctx* ctx, const float* d_x, int64_t n, int W, int hop, const double* d_window, int64_t num_frames,
                    void* d_out, int mode) {
    if (W <= 0 || hop <= 0 || num_frames <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "stft: bad window/hop/frames");
    urh_arena_reset(ctx);
    if (stft_smem_serves(W, num_frames, 0)) {
        double2* tw;
        URH_CHECK(urh_arena(ctx, (size_t)W, &tw));
        URH_LAUNCH(ctx, k_fft_twiddles, (unsigned)urh_div_up(W, 256), 256, 0, W, tw);
        return stft_r16(ctx, mode, W, d_x, n, hop, d_window, tw, num_frames, d_out, StftImage{});
    }
    // cuFFT with two kernels around it
    const int64_t max_batch = max((int64_t)1, ((int64_t)512 << 20) / ((int64_t)W * 16));
    const int64_t batch = min(num_frames, max_batch);
    double2* buf;
    URH_CHECK(urh_arena(ctx, (size_t)batch * W, &buf));
    const unsigned grid = (unsigned)min(urh_div_up(batch * W, 256), (int64_t)ctx->sm_count * 32);
    for (int64_t f0 = 0; f0 < num_frames; f0 += batch) {
        const int64_t nf = min(batch, num_frames - f0);
        URH_CHECK(ensure_plan(ctx, W, nf));
        URH_LAUNCH(ctx, k_stft_window, grid, 256, 0, (const float2*)d_x, n, W, hop, d_window, f0, nf, buf);
        URH_CUFFT(ctx, cufftExecZ2Z((cufftHandle)ctx->fft_plan, (cufftDoubleComplex*)buf, (cufftDoubleComplex*)buf, CUFFT_FORWARD));
        ctx->launches++;
        if (mode == 0) URH_LAUNCH(ctx, k_stft_scale, grid, 256, 0, buf, W, nf * W, (double2*)d_out + f0 * W);
        else URH_LAUNCH(ctx, k_stft_db, grid, 256, 0, buf, W, nf, (float*)d_out + f0 * W);
    }
    return URH_OK;
}

extern "C" int urh_stft(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window,
                        int64_t num_frames, double* d_out) {
    return stft_run(ctx, d_x, n, window_size, hop, d_window, num_frames, d_out, 0);
}

extern "C" int urh_spectrogram_db(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window,
                                  int64_t num_frames, float* d_out) {
    return stft_run(ctx, d_x, n, window_size, hop, d_window, num_frames, d_out, 1);
}

// ---- BGRA colormap look-up (Spectrogram.apply_bgra_lookup, Spectrogram.py:192-206; SURVEY 8f-4) --------------------------------
// out[c][r] = colormap[clip(int((L - 1) * ((data[r][c] - data_min) / (data_max - data_min))))]   (data.T: the image is transposed)
// float32 arithmetic in numpy's order (bgra_index): subtract, divide, multiply, truncate toward zero (astype(int)), np.take(mode="clip").
__global__ void k_bgra_lookup(const float* __restrict__ data, int64_t rows, int64_t cols, const uint32_t* __restrict__ colormap, int L,
                              float data_min, float range, int normalize, uint32_t* __restrict__ out) {
    __shared__ uint32_t s_map[1024];
    const bool in_smem = L <= 1024;
    if (in_smem)
        for (int i = threadIdx.x; i < L; i += blockDim.x) s_map[i] = colormap[i];
    __syncthreads();
    const int64_t total = rows * cols;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float scale = (float)(L - 1);
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int64_t c = idx / rows, r = idx - c * rows;   // output index (c, r) <- data[r][c]
        const int k = bgra_index(data[r * cols + c], data_min, range, scale, L, normalize);
        out[idx] = in_smem ? s_map[k] : colormap[k];
    }
}

// The reference's bounds are Python floats, which meet the float32 array as float32 (weak scalars): data_min on its own, and the
// range data_max - data_min formed in double first and rounded once.  Rounding the bounds before subtracting would round it twice.
static inline float bgra_range(double data_min, double data_max) { return (float)(data_max - data_min); }

extern "C" int urh_bgra_lookup(urh_ctx* ctx, const float* d_data, int64_t rows, int64_t cols, const uint8_t* d_colormap, int entries,
                               double data_min, double data_max, int normalize, uint8_t* d_out) {
    if (rows <= 0 || cols <= 0) return URH_OK;
    if (entries <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "bgra_lookup: empty colormap");
    const unsigned grid = (unsigned)min(urh_div_up(rows * cols, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_bgra_lookup, grid, 256, 0, d_data, rows, cols, (const uint32_t*)d_colormap, entries, (float)data_min,
               bgra_range(data_min, data_max), normalize, (uint32_t*)d_out);
    return URH_OK;
}

// ---- spectrogram images: STFT -> dB -> colormap in one launch (Spectrogram.create_spectrogram_image / create_image_segments) --------
// composed path: one chunk of dB rows (frames f0 .. f0 + nf - 1 of a segment with F frames) through the look-up into its place
// transpose = 0: out[r][f0 + f] (row pitch F) = lut(db[f][r]);  transpose = 1: out[f0 + f][r] = lut(db[f][W - 1 - r])
__global__ void k_bgra_place(const float* __restrict__ db, int64_t nf, int W, int64_t F, int64_t f0, const uint32_t* __restrict__ colormap,
                             int L, float data_min, float range, int transpose, uint32_t* __restrict__ out) {
    __shared__ uint32_t s_map[1024];
    const bool in_smem = L <= 1024;
    if (in_smem)
        for (int i = threadIdx.x; i < L; i += blockDim.x) s_map[i] = colormap[i];
    __syncthreads();
    const int64_t total = nf * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float scale = (float)(L - 1);
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        int64_t f, r, o;
        if (transpose) {
            f = idx / W; r = idx - f * W;
            o = (f0 + f) * W + r;
            r = W - 1 - r;
        } else {
            r = idx / nf; f = idx - r * nf;
            o = r * F + f0 + f;
        }
        const int k = bgra_index(db[f * W + r], data_min, range, scale, L, 1);
        out[o] = in_smem ? s_map[k] : colormap[k];
    }
}

extern "C" int urh_spectrogram_bgra(urh_ctx* ctx, const float* d_x, int64_t n, int window_size, int hop, const double* d_window,
                                    const int64_t* h_seg_start, const int64_t* h_seg_len, int nseg, const uint8_t* d_colormap, int entries,
                                    double data_min, double data_max, int transpose, uint8_t* d_out) {
    const int W = window_size;
    if (W <= 0 || hop <= 0 || nseg <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra: bad window/hop/segments");
    if (entries <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra: empty colormap");
    // per segment {start, end, frames, first block, first pixel}; frames as Spectrogram.stft counts them (short segments: one frame)
    std::vector<int64_t> seg((size_t)nseg * 5);
    int64_t blocks = 0, pixels = 0, max_frames = 0;
    for (int s = 0; s < nseg; s++) {
        const int64_t st = h_seg_start[s], len = h_seg_len[s];
        if (st < 0 || len < 0 || st + len > n) URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra: segment %d outside the capture", s);
        const int64_t F = len < W ? 1 : (len - W) / hop + 1;
        int64_t* g = &seg[(size_t)s * 5];
        g[0] = st; g[1] = st + len; g[2] = F; g[3] = blocks; g[4] = pixels;
        blocks += urh_div_up(F, STFT_IMG_FPB);
        pixels += F * W;
        max_frames = max(max_frames, F);
    }
    const float lo32 = (float)data_min, r32 = bgra_range(data_min, data_max);
    if (stft_smem_serves(W, blocks, entries)) {
        if (!ctx->img_tw) URH_CUDA(ctx, cudaMalloc(&ctx->img_tw, (size_t)4096 * sizeof(double2)));
        if (ctx->img_tw_n != W) {
            URH_LAUNCH(ctx, k_fft_twiddles, (unsigned)urh_div_up(W, 256), 256, 0, W, (double2*)ctx->img_tw);
            ctx->img_tw_n = W;
        }
        urh_arena_reset(ctx);
        int64_t* d_seg;
        URH_CHECK(urh_arena(ctx, seg.size(), &d_seg));
        URH_CUDA(ctx, cudaMemcpyAsync(d_seg, seg.data(), seg.size() * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
        const StftImage img{d_seg, nseg, (const uint32_t*)d_colormap, entries, lo32, r32, transpose ? 1 : 0};
        return stft_r16(ctx, 2, W, d_x, n, hop, d_window, (const double2*)ctx->img_tw, blocks, d_out, img);
    }
    // composed: the dB map of up to 256 MiB of frames at a time (stft_run), then its pixels into place
    const int64_t chunk = min(max_frames, max((int64_t)1, ((int64_t)256 << 20) / ((int64_t)W * 4)));
    float* db = nullptr;
    URH_CUDA(ctx, cudaMallocAsync((void**)&db, (size_t)chunk * W * sizeof(float), ctx->stream));
    int rc = URH_OK;
    for (int s = 0; s < nseg && rc == URH_OK; s++) {
        const int64_t* g = &seg[(size_t)s * 5];
        for (int64_t f0 = 0; f0 < g[2] && rc == URH_OK; f0 += chunk) {
            const int64_t nf = min(chunk, g[2] - f0), base = g[0] + f0 * hop;
            rc = stft_run(ctx, d_x + 2 * base, g[1] - base, W, hop, d_window, nf, db, 1);
            if (rc != URH_OK) break;
            const unsigned grid = (unsigned)min(urh_div_up(nf * W, 256), (int64_t)ctx->sm_count * 16);
            k_bgra_place<<<grid, 256, 0, ctx->stream>>>(db, nf, W, g[2], f0, (const uint32_t*)d_colormap, entries, lo32, r32,
                                                        transpose ? 1 : 0, (uint32_t*)d_out + g[4]);
            ctx->launches++;
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) {
                snprintf(ctx->err, sizeof(ctx->err), "spectrogram_bgra: k_bgra_place -> %s", cudaGetErrorString(e));
                rc = URH_ERR_CUDA;
            }
        }
    }
    cudaFreeAsync(db, ctx->stream);
    return rc;
}

// ---- host captures of any size through the windowed ring (stream_ring.cuh, DESIGN.md §4.11) ------------------------------------------
// A chunk is a run of whole frames [f0, f1) and uploads the samples they read; the window call is the one the sharded dB map runs
// (dist.py spectrogram_db_sharded), so every frame is the resident call's.
static int stft_stream(urh_ctx* ctx, const float* h_x, int64_t n, int W, int hop, const double* h_window, int64_t num_frames,
                       int64_t chunk_samples, int ring, void* h_out, int mode) {
    if (!h_x || !h_window || !h_out || W <= 0 || hop <= 0 || num_frames <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "stft_stream: bad arguments");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    const int entry = mode == 0 ? URH_FILTER_STFT : URH_FILTER_DB;
    std::vector<UrhWindow> win;
    URH_CHECK(urh_filter_windows(entry, n, num_frames, W, hop, chunk_samples, nullptr, nullptr, 0, win));
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, entry, n, num_frames, URH_DT_F32, W, hop, 0, chunk_samples, L));
    const double* d_window = (const double*)L.extra;
    URH_CUDA(ctx, cudaMemcpyAsync(L.extra, h_window, (size_t)W * 8, cudaMemcpyHostToDevice, ctx->stream));
    return stream_run(ctx, win, R, (const char*)h_x, 8, L.in, L.z.in_slot, true,
                      [&](int64_t, const UrhWindow& w, int s) {
                          return stft_run(ctx, (const float*)(L.in + s * L.z.in_slot), w.b - w.a, W, hop, d_window, w.k1 - w.k0,
                                          L.out + s * L.z.out_slot, mode);
                      },
                      contiguous_download(ctx, L.out, L.z.out_slot, (char*)h_out, (int64_t)W * (mode == 0 ? 16 : 4)));
}

extern "C" int urh_stft_stream(urh_ctx* ctx, const float* h_x, int64_t n, int window_size, int hop, const double* h_window, int64_t num_frames,
                               int64_t chunk_samples, int ring, double* h_out) {
    return stft_stream(ctx, h_x, n, window_size, hop, h_window, num_frames, chunk_samples, ring, h_out, 0);
}

extern "C" int urh_spectrogram_db_stream(urh_ctx* ctx, const float* h_x, int64_t n, int window_size, int hop, const double* h_window,
                                         int64_t num_frames, int64_t chunk_samples, int ring, float* h_out) {
    return stft_stream(ctx, h_x, n, window_size, hop, h_window, num_frames, chunk_samples, ring, h_out, 1);
}

// Images: a chunk is a group of whole segments (their images back to back, as the resident call writes them) or a run of frames of
// one long segment, rendered as a segment of its own; with transpose = 0 such a piece is the column band [W][f0:f1][4] of its image.
extern "C" int urh_spectrogram_bgra_stream(urh_ctx* ctx, const float* h_x, int64_t n, int window_size, int hop, const double* h_window,
                                           const int64_t* h_seg_start, const int64_t* h_seg_len, int nseg, const uint8_t* h_colormap,
                                           int entries, double data_min, double data_max, int transpose, int64_t chunk_samples, int ring,
                                           uint8_t* h_out) {
    const int W = window_size;
    if (!h_x || !h_window || !h_out || !h_colormap || W <= 0 || hop <= 0 || nseg <= 0)
        URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra_stream: bad window/hop/segments");
    if (entries <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra_stream: empty colormap");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    std::vector<UrhWindow> win;
    if (urh_filter_windows(URH_FILTER_IMAGES, n, 0, W, hop, chunk_samples, h_seg_start, h_seg_len, nseg, win) != URH_OK)
        URH_FAIL(ctx, URH_ERR_INVALID, "spectrogram_bgra_stream: a segment lies outside the capture");
    std::vector<int64_t> cum((size_t)nseg + 1, 0);   // frames before segment s
    for (int s = 0; s < nseg; s++) cum[s + 1] = cum[s] + (h_seg_len[s] < W ? 1 : (h_seg_len[s] - W) / hop + 1);
    StreamRing R;
    FilterRingLayout L;
    URH_CHECK(filter_ring_init(ctx, R, ring, URH_FILTER_IMAGES, n, cum[nseg], URH_DT_F32, W, hop, entries, chunk_samples, L));
    const double* d_window = (const double*)L.extra;
    const uint8_t* d_cmap = (const uint8_t*)(L.extra + r256((int64_t)W * 8));
    URH_CUDA(ctx, cudaMemcpyAsync(L.extra, h_window, (size_t)W * 8, cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync((void*)d_cmap, h_colormap, (size_t)entries * 4, cudaMemcpyHostToDevice, ctx->stream));
    // the segment holding frame k0, and whether the chunk lies within it.  Such a chunk (a run of its frames, or all of them) is
    // rendered as a segment of its own over the uploaded window, which holds exactly what its frames read and may end before the
    // segment does; its frame count from that window is the chunk's.  Other chunks are runs of whole segments.
    auto locate = [&](const UrhWindow& w, bool* piece) {
        const int s = (int)(std::upper_bound(cum.begin(), cum.end(), w.k0) - cum.begin()) - 1;
        *piece = w.k1 <= cum[s + 1];
        return s;
    };
    return stream_run(
        ctx, win, R, (const char*)h_x, 8, L.in, L.z.in_slot, true,
        [&](int64_t, const UrhWindow& w, int slot) {
            bool piece;
            const int s = locate(w, &piece);
            std::vector<int64_t> st, len;
            if (piece) {
                st.push_back(0);
                len.push_back(w.b - w.a);
            } else {
                for (int q = s; q < nseg && cum[q] < w.k1; q++) {
                    st.push_back(h_seg_start[q] - w.a);
                    len.push_back(h_seg_len[q]);
                }
            }
            return urh_spectrogram_bgra(ctx, (const float*)(L.in + slot * L.z.in_slot), w.b - w.a, W, hop, d_window, st.data(), len.data(),
                                        (int)st.size(), d_cmap, entries, data_min, data_max, transpose, (uint8_t*)(L.out + slot * L.z.out_slot));
        },
        [&](int64_t, const UrhWindow& w, int slot, cudaStream_t cp) {
            bool piece;
            const int s = locate(w, &piece);
            const char* src = L.out + slot * L.z.out_slot;
            const int64_t nf = w.k1 - w.k0;
            if (piece && !transpose) {   // rows of nf pixels into rows of the segment's F pixels (one copy when nf = F)
                const int64_t F = cum[s + 1] - cum[s];
                URH_CUDA(ctx, cudaMemcpy2DAsync(h_out + (cum[s] * W + (w.k0 - cum[s])) * 4, (size_t)F * 4, src, (size_t)nf * 4, (size_t)nf * 4,
                                                (size_t)W, cudaMemcpyDeviceToHost, cp));
            } else {
                URH_CUDA(ctx, cudaMemcpyAsync(h_out + w.k0 * W * 4, src, (size_t)(nf * W * 4), cudaMemcpyDeviceToHost, cp));
            }
            return URH_OK;
        });
}

// out[i] = x[start + i * step] (complex64 samples; Python slice semantics, step may be negative)
__global__ void k_gather_c64(const float2* __restrict__ x, int64_t start, int64_t step, int64_t count, float2* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) out[i] = x[start + i * step];
}

extern "C" int urh_gather_samples(urh_ctx* ctx, const float* d_x, int64_t n, int64_t start, int64_t step, int64_t count, float* d_out) {
    if (count <= 0) return URH_OK;
    const int64_t last = start + (count - 1) * step;
    if (start < 0 || start >= n || last < 0 || last >= n) URH_FAIL(ctx, URH_ERR_INVALID, "gather_samples: index outside the capture");
    const unsigned grid = (unsigned)min(urh_div_up(count, 256), (int64_t)ctx->sm_count * 16);
    URH_LAUNCH(ctx, k_gather_c64, grid, 256, 0, (const float2*)d_x, start, step, count, (float2*)d_out);
    return URH_OK;
}

// ---- FTA export records (Spectrogram.export_to_fta, Spectrogram.py:118-154) ---------------------------------------------------------
// The record array is [W][F][reps] of packed records {f8 f, u4 t[, f4 a]} (16 B with the amplitude, reps = 3; 12 B without, reps = 2):
// record (i, j) = {freqs[i], uint32(int(j * time_width)), dB_shift[j][i]}, each repeated reps times (numpy broadcasts the tuple).
// dB_shift[j][i] = db[j][W - 1 - i] (db is the fliplr'ed dB map).  A block covers 32 rows (bins) x 32 frames: it reads the dB tile
// along the bins and writes each row's 32 records, which are contiguous in the output, word by word.
template <int AMP>
__global__ void __launch_bounds__(256) k_fta_records(const float* __restrict__ db, int64_t F, int W, int64_t row0, int64_t nrows,
                                                     const double* __restrict__ freqs, double time_width, uint32_t* __restrict__ out) {
    constexpr int RW = AMP ? 4 : 3;            // 32-bit words per record
    constexpr int WPC = RW * (AMP ? 3 : 2);    // words per (i, j) cell
    __shared__ float s_a[32][33];              // [row][frame]
    const int64_t j0 = (int64_t)blockIdx.x * 32;
    const int64_t i0 = row0 + (int64_t)blockIdx.y * 32;
    if (AMP) {
        for (int e = threadIdx.x; e < 32 * 32; e += 256) {
            const int ii = e & 31, jj = e >> 5;
            const int64_t i = i0 + ii, j = j0 + jj;
            if (i < row0 + nrows && j < F) s_a[ii][jj] = db[j * W + (W - 1 - i)];
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < 32 * 32 * WPC; e += 256) {
        const int ii = e / (32 * WPC), rem = e - ii * (32 * WPC);
        const int jj = rem / WPC, q = (rem - jj * WPC) % RW;
        const int64_t i = i0 + ii, j = j0 + jj;
        if (i >= row0 + nrows || j >= F) continue;
        uint32_t v;
        if (q < 2) {
            const unsigned long long fb = (unsigned long long)__double_as_longlong(freqs[i]);
            v = q == 0 ? (uint32_t)fb : (uint32_t)(fb >> 32);
        } else if (q == 2) {
            v = (uint32_t)(long long)__dmul_rn((double)j, time_width);   // int(j * time_width); the host checked the range
        } else {
            v = __float_as_uint(s_a[ii][jj]);
        }
        out[((i - row0) * F + j) * WPC + (rem - jj * WPC)] = v;
    }
}

extern "C" int urh_fta_records(urh_ctx* ctx, const float* d_db, int64_t frames, int window_size, int64_t row0, int64_t nrows,
                               const double* d_freqs, double time_width, int include_amplitude, uint8_t* d_out, void* h_out) {
    const int W = window_size;
    if (W <= 0 || frames <= 0 || row0 < 0 || nrows < 0 || row0 + nrows > W) URH_FAIL(ctx, URH_ERR_INVALID, "fta_records: bad rows");
    if (nrows == 0) return URH_OK;
    const dim3 grid((unsigned)urh_div_up(frames, 32), (unsigned)urh_div_up(nrows, 32));
    if (grid.x >= (1u << 31) || grid.y > 65535) URH_FAIL(ctx, URH_ERR_INVALID, "fta_records: too many frames or rows");
    if (include_amplitude) URH_LAUNCH(ctx, k_fta_records<1>, grid, 256, 0, d_db, frames, W, row0, nrows, d_freqs, time_width, (uint32_t*)d_out);
    else URH_LAUNCH(ctx, k_fta_records<0>, grid, 256, 0, d_db, frames, W, row0, nrows, d_freqs, time_width, (uint32_t*)d_out);
    if (h_out) {
        const size_t bytes = (size_t)nrows * frames * (include_amplitude ? 48 : 24);
        URH_CUDA(ctx, cudaMemcpyAsync(h_out, d_out, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    }
    return URH_OK;
}
