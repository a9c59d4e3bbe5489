// detect_modulation on the GPU (SURVEY §8a row a10; AutoInterpretation.detect_modulation AutoInterpretation.py:151-208,
// Wavelet.cwt_haar Wavelet.py:15-43).  Everything at sample rate runs here; the handful of threshold comparisons that turn
// the features into "OOK" / "ASK" / "PSK" / "FSK" stay on the host (urh_b200/ainterpretation/AutoInterpretation.py).
//
//   data = data[|data| > 0]                         compaction (prefix sum)
//   data = data / |max(data)|                       np.max of a complex array is LEXICOGRAPHIC (real, then imag); float32 division
//   W1 = cwt_haar(data), W2 = cwt_haar(data/|data|) truncate to P = 2^floor(log2 n); FFT (numpy >= 2 keeps complex64 -> float32
//                                                   FFT: cuFFT C2C); x_hat * psi_hat in complex128, psi_hat the analytic Haar
//                                                   spectrum; inverse FFT in double (cuFFT Z2Z); crop 2*scale each side
//   var(|W1|), var(|W2|), var(median_filter(|W.|, k))
//   FSK test: |fftshift(fft(data[:P]))| -- the forward transform of W1 again: arg-max, the largest value >= 10 bins away
//             from it and the 19 values around it (enough to decide "one of the ten greatest is >= 10 bins away and >= 100").
// cuFFT is used for the FFTs only.  Parity: the float32 FFT differs from pocketfft in rounding, so features agree to ~1e-5
// relative; the tests compare features with that tolerance and the decisions on the golden captures exactly.
#include "common.cuh"
#include "tilescan.cuh"

#include <cufft.h>
#include <math.h>

#include <vector>

#define URH_CUFFT(ctx, call)                                                                                  \
    do {                                                                                                      \
        cufftResult r__ = (call);                                                                             \
        if (r__ != CUFFT_SUCCESS) {                                                                           \
            snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d: %s -> cufft error %d", __FILE__, __LINE__, #call, (int)r__); \
            return URH_ERR_CUDA;                                                                              \
        }                                                                                                     \
    } while (0)

// data[np.abs(data) > 0]: a NaN magnitude compares false, so (NaN, 0) is dropped while (inf, NaN), whose hypot is inf, stays
__device__ __forceinline__ bool urh_mod_keep(float2 v) { return hypotf(v.x, v.y) > 0.0f; }

// scan element: 1 for a kept sample; off[i] = kept samples before i (k_mod_compact's destination).  Scanned with 8 items per
// thread, as the per-row tables of bits.cu: faster than 16 on a per-sample table
struct ModKeepOffsets {
    const float2* x;
    int64_t* off;
    __device__ __forceinline__ int64_t load(int64_t i) const { return urh_mod_keep(x[i]) ? 1 : 0; }
    __device__ __forceinline__ void post(int64_t i, const int64_t& excl, const int64_t&) const { off[i] = excl; }
};

__global__ void k_mod_compact(const float2* __restrict__ x, int64_t n, const int64_t* __restrict__ off, float2* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float2 v = x[i];
        if (urh_mod_keep(v)) out[off[i]] = v;
    }
}

// lexicographic maximum (np.max on complex): block partials
__device__ __forceinline__ bool lex_greater(float2 a, float2 b) { return a.x > b.x || (a.x == b.x && a.y > b.y); }
__global__ void __launch_bounds__(256) k_mod_lexmax(const float2* __restrict__ x, int64_t n, float2* __restrict__ partial) {
    float2 best = make_float2(-INFINITY, -INFINITY);
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const float2 v = x[i];
        if (lex_greater(v, best)) best = v;
    }
    __shared__ float2 s[256];
    s[threadIdx.x] = best;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off && lex_greater(s[threadIdx.x + off], s[threadIdx.x])) s[threadIdx.x] = s[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}

// x1 = data / m (complex64 / float32), x2 = data / |data|; both truncated to P samples, batch layout [2][P]
__global__ void k_mod_normalise(const float2* __restrict__ x, int64_t P, float m, float2* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float2 v = x[i];
    const float2 a = make_float2(__fdiv_rn(v.x, m), __fdiv_rn(v.y, m));
    out[i] = a;
    const float mag = hypotf(a.x, a.y);   // np.abs(complex64) -> float32
    out[P + i] = make_float2(__fdiv_rn(a.x, mag), __fdiv_rn(a.y, mag));
}

// y = x_hat * psi_hat (complex128), psi_hat[k] = sqrt(2 pi s) * (1j * (-1 + exp(0.5j * s*omega_k))^2) / ((s*omega_k)/s), [0] -> /1
// XT = float2 (x_hat from the float32 transform) or double2 (complex128 input: in place on y)
template <typename XT>
__global__ void k_mod_psi_mul(const XT* __restrict__ xhat, int64_t P, int batch, double scale, double2* __restrict__ y) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const double f = 2.0 * M_PI / (double)P;
    const double omega = (k < P / 2) ? f * (double)k : f * ((double)k * -1.0);
    const double so = scale * omega;
    double den = so / scale;
    if (k == 0) den = 1.0;
    double sn, cs;
    sincos(0.5 * so, &sn, &cs);
    // e = -1 + exp(0.5j*so) = (cs - 1) + j sn;  e^2 = (er^2 - ei^2) + j (2 er ei);  1j * e^2 = (-2 er ei) + j (er^2 - ei^2)
    const double er = -1.0 + cs, ei = sn;
    const double sq_r = er * er - ei * ei, sq_i = er * ei + ei * er;
    const double amp = sqrt(2.0 * M_PI * scale);
    const double pr = amp * (-sq_i / den), pi_ = amp * (sq_r / den);
    for (int b = 0; b < batch; b++) {
        const XT xv = xhat[b * P + k];
        const double xr = (double)xv.x, xi = (double)xv.y;
        y[b * P + k] = make_double2(xr * pr - xi * pi_, xr * pi_ + xi * pr);
    }
}

__global__ void k_mod_crop_scale(const double2* __restrict__ y, int64_t P, int64_t crop, int64_t L, double2* __restrict__ out) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= L) return;
    const double inv = 1.0 / (double)P;
    const double2 v = y[j + crop];
    out[j] = make_double2(v.x * inv, v.y * inv);
}

__global__ void k_mod_dup(const void* __restrict__ x, int is_c128, int64_t P, float2* __restrict__ xf, double2* __restrict__ xd) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (is_c128) { const double2 v = ((const double2*)x)[i]; xd[i] = v; xd[P + i] = v; }
    else { const float2 v = ((const float2*)x)[i]; xf[i] = v; xf[P + i] = v; }
}

// |W| after the 1/P of numpy's ifft, cropped: mag[b][j] = |y[b][j + crop]| / P, j < L
__global__ void k_mod_mag(const double2* __restrict__ y, int64_t P, int64_t crop, int64_t L, double* __restrict__ mag) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= L) return;
    const double inv = 1.0 / (double)P;
    for (int b = 0; b < 2; b++) {
        const double2 v = y[b * P + j + crop];
        mag[b * L + j] = hypot(v.x * inv, v.y * inv);
    }
}

// sum and sum of squared deviations from `mean` (call with mean = 0 for the plain sum), block partials
template <typename T>
__global__ void __launch_bounds__(256) k_mod_moments(const T* __restrict__ x, int64_t n, double mean, double* __restrict__ partial) {
    double s = 0.0, q = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        const double d = (double)x[i] - mean;
        s += d;
        q += d * d;
    }
    __shared__ double ss[256], sq[256];
    ss[threadIdx.x] = s; sq[threadIdx.x] = q;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) { ss[threadIdx.x] += ss[threadIdx.x + off]; sq[threadIdx.x] += sq[threadIdx.x + off]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { partial[2 * blockIdx.x] = ss[0]; partial[2 * blockIdx.x + 1] = sq[0]; }
}

// median_filter (auto_interpretation.pyx:211-240): window [i, i+k) truncated at the end, float32 values, sorted[k'//2]
__global__ void k_mod_median(const double* __restrict__ x, int64_t n, int k, float* __restrict__ out) {
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

// |fftshift(x_hat)| (float32 hypot) and block partials of (max value, index); pass far_from >= 0 to skip |i - far_from| < 10
__global__ void __launch_bounds__(256) k_mod_specmax(const float2* __restrict__ xhat, int64_t P, int64_t far_from, float* __restrict__ pv,
                                                    int64_t* __restrict__ pi_) {
    float best = -1.0f;
    int64_t bi = -1;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < P; i += (int64_t)gridDim.x * 256) {
        if (far_from >= 0 && llabs(i - far_from) < 10) continue;
        const float2 v = xhat[(i + P / 2) % P];   // fftshift: shifted[i] = x_hat[(i + P/2) mod P] for even P (P = 1 -> itself)
        const float a = hypotf(v.x, v.y);
        if (a > best || (a == best && i > bi)) { best = a; bi = i; }   // ties: the later index (argsort()[::-1] order for equal keys is unspecified)
    }
    __shared__ float sv[256];
    __shared__ int64_t si[256];
    sv[threadIdx.x] = best; si[threadIdx.x] = bi;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
            const float a = sv[threadIdx.x + off];
            const int64_t b = si[threadIdx.x + off];
            if (a > sv[threadIdx.x] || (a == sv[threadIdx.x] && b > si[threadIdx.x])) { sv[threadIdx.x] = a; si[threadIdx.x] = b; }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { pv[blockIdx.x] = sv[0]; pi_[blockIdx.x] = si[0]; }
}

__global__ void k_mod_near(const float2* __restrict__ xhat, int64_t P, int64_t g, float* __restrict__ out19) {
    const int j = threadIdx.x;   // 0..18 -> index g - 9 + j
    if (j >= 19) return;
    const int64_t i = g - 9 + j;
    float a = -1.0f;
    if (i >= 0 && i < P) {
        const float2 v = xhat[(i + P / 2) % P];
        a = hypotf(v.x, v.y);
    }
    out19[j] = a;
}

static int moments(urh_ctx* ctx, const void* d_x, bool is_f32, int64_t n, double* h_var) {
    // np.var: mean of squared deviations from the mean (two passes, double)
    const int nb = (int)min((int64_t)ctx->sm_count * 4, urh_div_up(n, 256));
    double* partial;
    URH_CHECK(urh_arena(ctx, (size_t)2 * nb + 2, &partial));
    std::vector<double> h((size_t)2 * nb);
    auto pass = [&](double mean, double* s, double* q) -> int {
        if (is_f32) URH_LAUNCH(ctx, k_mod_moments<float>, nb, 256, 0, (const float*)d_x, n, mean, partial);
        else URH_LAUNCH(ctx, k_mod_moments<double>, nb, 256, 0, (const double*)d_x, n, mean, partial);
        URH_CUDA(ctx, cudaMemcpyAsync(h.data(), partial, h.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *s = 0.0; *q = 0.0;
        for (int b = 0; b < nb; b++) { *s += h[2 * b]; *q += h[2 * b + 1]; }
        return URH_OK;
    };
    double s, q;
    URH_CHECK(pass(0.0, &s, &q));
    const double mean = s / (double)n;
    URH_CHECK(pass(mean, &s, &q));
    *h_var = q / (double)n;
    return URH_OK;
}

static int mod_plan(urh_ctx* ctx, int which, cufftType type, int64_t P) {
    if (ctx->mod_plan_valid[which] && ctx->mod_plan_n[which] == P) return URH_OK;
    if (ctx->mod_plan_valid[which]) {
        cufftDestroy((cufftHandle)ctx->mod_plan[which]);
        ctx->mod_plan_valid[which] = 0;
    }
    cufftHandle plan;
    int nfft[1] = {(int)P};
    URH_CUFFT(ctx, cufftPlanMany(&plan, 1, nfft, nullptr, 1, (int)P, nullptr, 1, (int)P, type, 2));
    URH_CUFFT(ctx, cufftSetStream(plan, ctx->stream));
    ctx->mod_plan[which] = (int)plan;
    ctx->mod_plan_n[which] = P;
    ctx->mod_plan_valid[which] = 1;
    return URH_OK;
}

// d_data: complex64[n] on the device (one message).  h_feat[8] = {n_nonzero, P, L, var_mag, var_norm_mag, var_filtered_mag,
// var_filtered_norm_mag, |max|}; h_spec[22] = {argmax index g, value, far index, far value (-1: none), 19 values around g
// (index g-9 .. g+9, -1 outside the spectrum)} -- all of the shifted float32 magnitude spectrum of the first P samples.
// L == 0 (fewer than 4*scale + 1 usable samples) or n_nonzero == 0: no features (detect_modulation returns None).
extern "C" int urh_modulation_features(urh_ctx* ctx, const float* d_data, int64_t n, int wavelet_scale, int median_k, double* h_feat,
                                       double* h_spec) {
    for (int i = 0; i < 8; i++) h_feat[i] = 0.0;
    for (int i = 0; i < 23; i++) h_spec[i] = -1.0;
    if (n <= 0) return URH_OK;
    if (wavelet_scale < 1 || median_k < 1 || median_k > 64) URH_FAIL(ctx, URH_ERR_INVALID, "wavelet_scale >= 1 and 1 <= median k <= 64 required");
    urh_arena_reset(ctx);
    const float2* x = (const float2*)d_data;
    int64_t *off, *d_cnt;
    URH_CHECK(urh_arena(ctx, (size_t)n, &off));
    URH_CHECK(urh_arena(ctx, 4, &d_cnt));
    const unsigned g = (unsigned)urh_div_up(n, 256);
    ModKeepOffsets fk;
    fk.x = x; fk.off = off;
    URH_CHECK((urhts::scan<int64_t, urhts::AddI64, ModKeepOffsets, 8>(ctx, n, (int64_t)0, urhts::AddI64(), fk, d_cnt)));
    int64_t nz = 0;
    URH_CHECK(urh_read_i64(ctx, d_cnt, 1, &nz));
    h_feat[0] = (double)nz;
    if (nz == 0 || n - nz > 3) return URH_OK;   // None / "OOK" without looking further (AutoInterpretation.py:154-159)
    float2* data;
    URH_CHECK(urh_arena(ctx, (size_t)nz, &data));
    URH_LAUNCH(ctx, k_mod_compact, g, 256, 0, x, n, off, data);
    // |max(data)|: lexicographic maximum, then float32 hypot
    const int nb = (int)min((int64_t)ctx->sm_count * 2, urh_div_up(nz, 256));
    float2* pmax;
    URH_CHECK(urh_arena(ctx, (size_t)nb, &pmax));
    URH_LAUNCH(ctx, k_mod_lexmax, nb, 256, 0, data, nz, pmax);
    std::vector<float2> hmax((size_t)nb);
    URH_CUDA(ctx, cudaMemcpyAsync(hmax.data(), pmax, (size_t)nb * sizeof(float2), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    float2 best = hmax[0];
    for (int b = 1; b < nb; b++)
        if (hmax[b].x > best.x || (hmax[b].x == best.x && hmax[b].y > best.y)) best = hmax[b];
    const float m = hypotf(best.x, best.y);
    h_feat[7] = (double)m;
    int64_t P = 1;
    while (P * 2 <= nz) P *= 2;
    const int64_t crop = 2 * (int64_t)wavelet_scale;
    const int64_t L = P - 2 * crop;   // len(W[2s : -2s])
    h_feat[1] = (double)P;
    h_feat[2] = (double)(L > 0 ? L : 0);
    if (L <= 0) return URH_OK;
    if (P > ((int64_t)1 << 27)) URH_FAIL(ctx, URH_ERR_INVALID, "message too long for the wavelet FFT");
    float2* xn;
    double2* y;
    double* mag;
    float* filt;
    URH_CHECK(urh_arena(ctx, (size_t)2 * P, &xn));
    URH_CHECK(urh_arena(ctx, (size_t)2 * P, &y));
    URH_CHECK(urh_arena(ctx, (size_t)2 * L, &mag));
    URH_CHECK(urh_arena(ctx, (size_t)L, &filt));
    const unsigned gp = (unsigned)urh_div_up(P, 256);
    URH_LAUNCH(ctx, k_mod_normalise, gp, 256, 0, (const float2*)data, P, m, xn);
    URH_CHECK(mod_plan(ctx, 0, CUFFT_C2C, P));
    URH_CHECK(mod_plan(ctx, 1, CUFFT_Z2Z, P));
    URH_CUFFT(ctx, cufftExecC2C((cufftHandle)ctx->mod_plan[0], (cufftComplex*)xn, (cufftComplex*)xn, CUFFT_FORWARD));
    URH_LAUNCH(ctx, k_mod_psi_mul<float2>, gp, 256, 0, (const float2*)xn, P, 2, (double)wavelet_scale, y);
    URH_CUFFT(ctx, cufftExecZ2Z((cufftHandle)ctx->mod_plan[1], (cufftDoubleComplex*)y, (cufftDoubleComplex*)y, CUFFT_INVERSE));
    URH_LAUNCH(ctx, k_mod_mag, (unsigned)urh_div_up(L, 256), 256, 0, (const double2*)y, P, crop, L, mag);
    URH_CHECK(moments(ctx, mag, false, L, &h_feat[3]));
    URH_CHECK(moments(ctx, mag + L, false, L, &h_feat[4]));
    for (int b = 0; b < 2; b++) {
        URH_LAUNCH(ctx, k_mod_median, (unsigned)urh_div_up(L, 128), 128, 0, (const double*)(mag + b * L), L, median_k, filt);
        URH_CHECK(moments(ctx, filt, true, L, &h_feat[5 + b]));
    }
    // spectrum features of the first transform (x_hat of data[:P] is still in xn[0..P))
    {
        const int sb = (int)min((int64_t)ctx->sm_count * 2, urh_div_up(P, 256));
        float* pv;
        int64_t* pidx;
        float* near19;
        URH_CHECK(urh_arena(ctx, (size_t)sb, &pv));
        URH_CHECK(urh_arena(ctx, (size_t)sb, &pidx));
        URH_CHECK(urh_arena(ctx, 32, &near19));
        std::vector<float> hv((size_t)sb);
        std::vector<int64_t> hi((size_t)sb);
        auto specmax = [&](int64_t far_from, double* idx, double* val) -> int {
            URH_LAUNCH(ctx, k_mod_specmax, sb, 256, 0, (const float2*)xn, P, far_from, pv, pidx);
            URH_CUDA(ctx, cudaMemcpyAsync(hv.data(), pv, (size_t)sb * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
            URH_CUDA(ctx, cudaMemcpyAsync(hi.data(), pidx, (size_t)sb * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
            URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            float bv = -1.0f;
            int64_t bi = -1;
            for (int b = 0; b < sb; b++)
                if (hi[b] >= 0 && (hv[b] > bv || (hv[b] == bv && hi[b] > bi))) { bv = hv[b]; bi = hi[b]; }
            *idx = (double)bi;
            *val = (double)bv;
            return URH_OK;
        };
        URH_CHECK(specmax(-1, &h_spec[0], &h_spec[1]));
        URH_CHECK(specmax((int64_t)h_spec[0], &h_spec[2], &h_spec[3]));
        URH_LAUNCH(ctx, k_mod_near, 1, 32, 0, (const float2*)xn, P, (int64_t)h_spec[0], near19);
        float hn[19];
        URH_CUDA(ctx, cudaMemcpyAsync(hn, near19, sizeof(hn), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int j = 0; j < 19; j++) h_spec[4 + j] = (double)hn[j];
    }
    return URH_OK;
}

// Wavelet.cwt_haar (Wavelet.py:15-43) of one array: complex64 input -> float32 forward transform (as numpy >= 2 does),
// complex128 input -> double.  d_out: complex128[P - 4*scale], P = 2^floor(log2 n); *out_len = that length (0: nothing written).
extern "C" int urh_cwt_haar(urh_ctx* ctx, const void* d_x, int is_c128, int64_t n, int scale, double* d_out, int64_t* out_len) {
    if (!out_len) return URH_ERR_INVALID;
    *out_len = 0;
    if (n <= 0) return URH_OK;
    if (scale < 1) URH_FAIL(ctx, URH_ERR_INVALID, "scale >= 1 required");
    urh_arena_reset(ctx);
    int64_t P = 1;
    while (P * 2 <= n) P *= 2;
    const int64_t crop = 2 * (int64_t)scale, L = P - 2 * crop;
    if (L <= 0) return URH_OK;
    if (P > ((int64_t)1 << 27)) URH_FAIL(ctx, URH_ERR_INVALID, "array too long for the wavelet FFT");
    float2* xf = nullptr;
    double2* y;
    URH_CHECK(urh_arena(ctx, (size_t)2 * P, &y));
    if (!is_c128) URH_CHECK(urh_arena(ctx, (size_t)2 * P, &xf));
    const unsigned gp = (unsigned)urh_div_up(P, 256);
    URH_LAUNCH(ctx, k_mod_dup, gp, 256, 0, d_x, is_c128, P, xf, y);   // the plans are batch-2 (detect_modulation's shape)
    URH_CHECK(mod_plan(ctx, 1, CUFFT_Z2Z, P));
    if (is_c128) {
        URH_CUFFT(ctx, cufftExecZ2Z((cufftHandle)ctx->mod_plan[1], (cufftDoubleComplex*)y, (cufftDoubleComplex*)y, CUFFT_FORWARD));
        URH_LAUNCH(ctx, k_mod_psi_mul<double2>, gp, 256, 0, (const double2*)y, P, 1, (double)scale, y);
    } else {
        URH_CHECK(mod_plan(ctx, 0, CUFFT_C2C, P));
        URH_CUFFT(ctx, cufftExecC2C((cufftHandle)ctx->mod_plan[0], (cufftComplex*)xf, (cufftComplex*)xf, CUFFT_FORWARD));
        URH_LAUNCH(ctx, k_mod_psi_mul<float2>, gp, 256, 0, (const float2*)xf, P, 1, (double)scale, y);
    }
    URH_CUFFT(ctx, cufftExecZ2Z((cufftHandle)ctx->mod_plan[1], (cufftDoubleComplex*)y, (cufftDoubleComplex*)y, CUFFT_INVERSE));
    URH_LAUNCH(ctx, k_mod_crop_scale, (unsigned)urh_div_up(L, 256), 256, 0, (const double2*)y, P, crop, L, (double2*)d_out);
    *out_len = L;
    return URH_OK;
}

void urh_release_mod_plans(urh_ctx* ctx) {
    for (int i = 0; i < 2; i++)
        if (ctx->mod_plan_valid[i]) {
            cufftDestroy((cufftHandle)ctx->mod_plan[i]);
            ctx->mod_plan_valid[i] = 0;
        }
}

// arg-max of |fft(x)| (float32 transform and magnitudes, as numpy computes them for complex64 input); first index on ties.
__global__ void __launch_bounds__(256) k_mod_argmax_first(const float2* __restrict__ xhat, int64_t P, float* __restrict__ pv, int64_t* __restrict__ pi_) {
    float best = -1.0f;
    int64_t bi = -1;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < P; i += (int64_t)gridDim.x * 256) {
        const float2 v = xhat[i];
        const float a = hypotf(v.x, v.y);
        if (a > best) { best = a; bi = i; }   // ascending i per thread: keeps the first
    }
    __shared__ float sv[256];
    __shared__ int64_t si[256];
    sv[threadIdx.x] = best; si[threadIdx.x] = bi;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
            const float a = sv[threadIdx.x + off];
            const int64_t b = si[threadIdx.x + off];
            if (b >= 0 && (a > sv[threadIdx.x] || (a == sv[threadIdx.x] && b < si[threadIdx.x]) || si[threadIdx.x] < 0)) { sv[threadIdx.x] = a; si[threadIdx.x] = b; }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { pv[blockIdx.x] = sv[0]; pi_[blockIdx.x] = si[0]; }
}

// Signal.estimate_frequency (Signal.py:578-601): index of the strongest bin of fft(x[0:P]), P = 2^floor(log2 n).
// *h_index in [0, P); the caller maps it through np.fft.fftfreq.  *h_P = P (0: n == 0).
extern "C" int urh_fft_argmax(urh_ctx* ctx, const float* d_x, int64_t n, int64_t* h_index, int64_t* h_P) {
    if (!h_index || !h_P) return URH_ERR_INVALID;
    *h_index = 0; *h_P = 0;
    if (n <= 0) return URH_OK;
    urh_arena_reset(ctx);
    int64_t P = 1;
    while (P * 2 <= n) P *= 2;
    if (P > ((int64_t)1 << 27)) URH_FAIL(ctx, URH_ERR_INVALID, "window too long for the FFT");
    float2* xf;
    double2* unused = nullptr;
    URH_CHECK(urh_arena(ctx, (size_t)2 * P, &xf));
    URH_LAUNCH(ctx, k_mod_dup, (unsigned)urh_div_up(P, 256), 256, 0, (const void*)d_x, 0, P, xf, unused);
    URH_CHECK(mod_plan(ctx, 0, CUFFT_C2C, P));
    URH_CUFFT(ctx, cufftExecC2C((cufftHandle)ctx->mod_plan[0], (cufftComplex*)xf, (cufftComplex*)xf, CUFFT_FORWARD));
    const int sb = (int)min((int64_t)ctx->sm_count * 2, urh_div_up(P, 256));
    float* pv;
    int64_t* pidx;
    URH_CHECK(urh_arena(ctx, (size_t)sb, &pv));
    URH_CHECK(urh_arena(ctx, (size_t)sb, &pidx));
    URH_LAUNCH(ctx, k_mod_argmax_first, sb, 256, 0, (const float2*)xf, P, pv, pidx);
    std::vector<float> hv((size_t)sb);
    std::vector<int64_t> hi((size_t)sb);
    URH_CUDA(ctx, cudaMemcpyAsync(hv.data(), pv, (size_t)sb * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(hi.data(), pidx, (size_t)sb * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    float bv = -1.0f;
    int64_t bi = -1;
    for (int b = 0; b < sb; b++)
        if (hi[b] >= 0 && (hv[b] > bv || (hv[b] == bv && hi[b] < bi) || bi < 0)) { bv = hv[b]; bi = hi[b]; }
    *h_index = bi < 0 ? 0 : bi;
    *h_P = P;
    return URH_OK;
}
