// PSK demodulation: Costas loop (reference: signal_functions.pyx:252-330, costa_demod).
//
// The loop is a nonlinear serial recurrence over ALL non-noise samples (costa_freq / costa_phase carried
// sample to sample, frozen on noise samples) — there is no exact parallel form (SURVEY H2).  This kernel
// keeps the recurrence on one lane and uses the rest of the warp as a software pipeline: the warp stages
// the next chunk of samples (converted, noise-gated, scaled) into shared memory and writes the previous
// chunk of results back with coalesced stores, so the serial lane never waits on global memory.
#include "dense.cuh"
#include "glibc_sincosf.h"

#include <math.h>

#define COSTAS_CHUNK 2048

struct CostasParams {
    float noise_sqrd, alpha, beta, scale, shift;
    int order;
};

// st_in (NULL: the loop's initial state {0, 1.5}) / st_out: {freq, phase} before / after the n samples on the device (the ring chunks
// of a streamed capture carry the state this way); cap_start: sample 0 is the capture's first (the reference skips it)
template <int DT>
__global__ void __launch_bounds__(32) k_costas(const void* __restrict__ iq, int64_t n, CostasParams P,
                                               float* __restrict__ out, int write_first, const float* __restrict__ st_in,
                                               float* __restrict__ st_out, int cap_start) {
    __shared__ float s_re[2][COSTAS_CHUNK];
    __shared__ float s_im[2][COSTAS_CHUNK];
    __shared__ float s_out[2][COSTAS_CHUNK];
    typedef typename UrhElem<DT>::type E;
    const E* p = (const E*)iq;
    const int lane = threadIdx.x;
    float freq = 0.0f, phase = 1.5f;
    if (st_in) {
        freq = st_in[0];
        phase = st_in[1];
    }
    const double two_pi_d = 2 * M_PI;  // the reference compares/adjusts the float phase in double
    const int64_t nchunks = (n + COSTAS_CHUNK - 1) / COSTAS_CHUNK;

    auto stage = [&](int64_t c, int buf) {
        const int64_t base = c * COSTAS_CHUNK;
        for (int j = lane; j < COSTAS_CHUNK; j += 32) {
            const int64_t i = base + j;
            float re = 0.f, im = 0.f;
            if (i < n) {
                re = (float)p[2 * i];
                im = (float)p[2 * i + 1];
            }
            s_re[buf][j] = re;
            s_im[buf][j] = im;
        }
    };
    stage(0, 0);
    __syncwarp();
    for (int64_t c = 0; c < nchunks; c++) {
        const int buf = (int)(c & 1);
        const int64_t base = c * COSTAS_CHUNK;
        const int len = (int)((n - base) < COSTAS_CHUNK ? (n - base) : COSTAS_CHUNK);
        if (lane == 0) {
            for (int j = 0; j < len; j++) {
                if (cap_start && base + j == 0) continue;  // the reference loop starts at i = 1 (pyx:289)
                const float re = s_re[buf][j], im = s_im[buf][j];
                if (__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)) <= P.noise_sqrd) {
                    s_out[buf][j] = -4.0f;
                    continue;
                }
                const float rf = __fdiv_rn(__fadd_rn(re, P.shift), P.scale);
                const float jf = __fdiv_rn(__fadd_rn(im, P.shift), P.scale);
                // current_sample = rf + 1j*jf  (std::complex<float> arithmetic, as in urh_demod_one)
                const float cs_r = __fadd_rn(rf, __fsub_rn(__fmul_rn(0.0f, jf), 0.0f));
                const float cs_i = __fadd_rn(0.0f, __fadd_rn(0.0f, jf));
                // glibc 2.39 sinf/cosf restated bit-for-bit (glibc_sincosf.h); |phase| <= 2*pi + 2 < 120 always
                float sn, cn;
                int sc_ok;
                urh_glibc_sincosf(-phase, &sn, &cn, &sc_ok);
                if (!sc_ok) sincosf(-phase, &sn, &cn);
                // nco_out = cosf(-phase) + 1j*sinf(-phase)
                const float nr = __fadd_rn(cn, __fsub_rn(__fmul_rn(0.0f, sn), 0.0f));
                const float ni = __fadd_rn(0.0f, __fadd_rn(0.0f, sn));
                // nco_times_sample = nco_out * current_sample: GCC's complex product, Annex G recovery included (an
                // infinite imaginary part of the sample gives an infinite product, not NaN); 1j*jf and 1j*sin above never
                // reach the recovery (only one of their parts can be NaN unless jf is NaN, and then no operand is infinite)
                float xr, xi;
                urh_cmulf(nr, ni, cs_r, cs_i, xr, xi);
                float err;
                if (P.order == 2) err = __fmul_rn(xi, xr);
                else {
                    const float f1 = xr > 0.0f ? 1.0f : -1.0f;
                    const float f2 = xi > 0.0f ? 1.0f : -1.0f;
                    err = __fsub_rn(__fmul_rn(f1, xi), __fmul_rn(f2, xr));
                }
                err = err < -1.0f ? -1.0f : (err > 1.0f ? 1.0f : err);
                freq = __fadd_rn(freq, __fmul_rn(P.beta, err));
                phase = __fadd_rn(phase, __fadd_rn(freq, __fmul_rn(P.alpha, err)));
                // float phase compared / adjusted against the double constant 2*M_PI (pyx:318-321)
                while ((double)phase > two_pi_d) phase = (float)((double)phase - two_pi_d);
                while ((double)phase < -two_pi_d) phase = (float)((double)phase + two_pi_d);
                freq = freq < -1.0f ? -1.0f : (freq > 1.0f ? 1.0f : freq);
                // order 4: (2.0 * re) + im is evaluated in double and stored to float (pyx:328)
                s_out[buf][j] = (P.order == 2) ? xr : (float)(2.0 * (double)xr + (double)xi);
            }
        } else if (c + 1 < nchunks) {
            // lanes 1..31 stage the next chunk while lane 0 runs the recurrence
            const int64_t nb = (c + 1) * COSTAS_CHUNK;
            for (int j = lane - 1; j < COSTAS_CHUNK; j += 31) {
                const int64_t i = nb + j;
                float re = 0.f, im = 0.f;
                if (i < n) {
                    re = (float)p[2 * i];
                    im = (float)p[2 * i + 1];
                }
                s_re[buf ^ 1][j] = re;
                s_im[buf ^ 1][j] = im;
            }
        }
        __syncwarp();
        for (int j = lane; j < len; j += 32) {
            const bool first = cap_start && base + j == 0;
            if (first && !write_first) continue;
            out[base + j] = first ? 0.0f : s_out[buf][j];
        }
        __syncwarp();
    }
    if (lane == 0 && st_out) {
        st_out[0] = freq;
        st_out[1] = phase;
    }
}

int urh_costas_demod_serial(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_sqrd, int loop_order,
                            float bandwidth, float* d_out, const float* d_st_in, float* d_st_out, int cap_start) {
    // signal_functions.pyx:252-287
    CostasParams P;
    const float damping = (float)(sqrt(2.0) / 2.0);
    // alpha/beta: the reference evaluates these in double (float operands promoted by the double literals)
    // generated C: ((double)((4.0 * damping) * bandwidth)) / ((1.0 + ((2.0 * damping) * bandwidth)) + (bandwidth * bandwidth))
    // with float damping/bandwidth: the products with double literals are double, bandwidth*bandwidth is float.
    const double bw = (double)bandwidth, dm = (double)damping;
    volatile float bw2f = bandwidth * bandwidth;
    const double den = (1.0 + ((2.0 * dm) * bw)) + (double)bw2f;
    P.alpha = (float)(((4.0 * dm) * bw) / den);
    P.beta = (float)(((4.0 * bw) * bw) / den);
    P.noise_sqrd = noise_sqrd;
    switch (dtype) {
        case URH_DT_I8: P.scale = 127.5f; P.shift = 0.5f; break;
        case URH_DT_U8: P.scale = 127.5f; P.shift = -127.5f; break;
        case URH_DT_I16: P.scale = 32767.5f; P.shift = 0.5f; break;
        case URH_DT_U16: P.scale = 65535.0f; P.shift = -32767.5f; break;
        case URH_DT_F32: P.scale = 1.0f; P.shift = 0.0f; break;
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    }
    P.order = loop_order > 4 ? 4 : loop_order;  // pyx:285-287
    // the speculative path's diagnostics describe the last PSK call: this one has no chunks, chains or stitch (segs = 0)
    for (int i = 0; i < 3; i++) ctx->costas_stats[i] = 0;
    ctx->costas_redone = 0;
    for (int i = 0; i < 4; i++) ctx->costas_stitch[i] = 0;
    // result[0] is uninitialised in the reference (np.empty, pyx:265); we define it as 0.
    switch (dtype) {
        case URH_DT_I8: URH_LAUNCH(ctx, k_costas<URH_DT_I8>, 1, 32, 0, d_iq, n, P, d_out, 1, d_st_in, d_st_out, cap_start); break;
        case URH_DT_U8: URH_LAUNCH(ctx, k_costas<URH_DT_U8>, 1, 32, 0, d_iq, n, P, d_out, 1, d_st_in, d_st_out, cap_start); break;
        case URH_DT_I16: URH_LAUNCH(ctx, k_costas<URH_DT_I16>, 1, 32, 0, d_iq, n, P, d_out, 1, d_st_in, d_st_out, cap_start); break;
        case URH_DT_U16: URH_LAUNCH(ctx, k_costas<URH_DT_U16>, 1, 32, 0, d_iq, n, P, d_out, 1, d_st_in, d_st_out, cap_start); break;
        default: URH_LAUNCH(ctx, k_costas<URH_DT_F32>, 1, 32, 0, d_iq, n, P, d_out, 1, d_st_in, d_st_out, cap_start); break;
    }
    return URH_OK;
}
