// Modulator forward path: ASK / FSK / PSK / OQPSK / GFSK (reference: signal_functions.pyx:56-243,
// modulate_c / __modulate / get_gauss_filtered_freqs_phases / gauss_fir / get_oqpsk_bits).
//
// A call modulates a BATCH of messages that share one parameter set (how every reference caller uses it:
// Modulator.modulate per message from modulate_messages / ContinuousModulator / the simulator, always start=0
// — SURVEY §3.3, H4).  Per message:
//   * FSK: the per-symbol phase corrections are a float32-rounded serial recurrence over the symbols
//     (pyx:121-137) -> one thread per message walks them (double fmod, exactly as the C code does);
//   * GFSK: per-sample frequencies = Gaussian-filtered symbol frequencies (np.convolve 'same'), then a
//     float32-rounded serial phase recurrence over all samples (pyx:220-224) -> one thread per message;
//   * then every sample is independent: t = (float)(i+start)/sample_rate, arg = (float)(2*pi*f*t + phi + corr)
//     evaluated in double, I/Q = a*cosf(arg), a*sinf(arg) with glibc's sinf/cosf restated bit-for-bit
//     (glibc_sincosf.h) and C truncation to the integer output types.
// Bit-exact for ASK/FSK/PSK/OQPSK.  GFSK is tolerance-parity: numpy's float32 convolution runs in OpenBLAS
// sdot, whose summation order depends on the host CPU (DESIGN.md).
#include "common.cuh"
#include "glibc_sincosf.h"

#include <math.h>

struct ModParams {
    uint32_t sps;
    int mod_type;
    int bps;
    float a, f, phi, sample_rate;
    uint32_t start;
    int out_dtype;
    int nparams;
    float params[256];
};

__device__ __forceinline__ uint32_t symbol_index(const uint8_t* bits, int64_t s, int bps) {
    // bit_array_to_number(bits, end=(s+1)*bps, start=s*bps): MSB first (util.pyx:50-61)
    uint32_t r = 0;
    for (int b = 0; b < bps; b++) r = r * 2u + (uint32_t)bits[s * bps + b];
    return r;
}

// fmod(v, 2 pi) exactly as C's fmod (sign of v, |result| < 2 pi), without the generic bit-by-bit long division: one estimate of the
// quotient and an FMA.  Exact: v and q * 2pi are multiples of ulp(2 pi) = 2^-50, so the true remainder v - q * 2pi (< 8) is a
// double and fma(-q, 2pi, |v|) returns it unrounded; an estimate that is off by one is corrected from the remainder's sign / size.
__device__ __forceinline__ double urh_fmod_2pi(double v) {
    const double y = 2.0 * M_PI;
    const double av = fabs(v);
    if (!(av < 1.0e15)) return fmod(v, y);   // huge, inf, nan: the library routine
    if (av < y) return v;
    double q = trunc(av * (1.0 / y));
    double r = fma(-q, y, av);
    while (r < 0.0) { q -= 1.0; r = fma(-q, y, av); }
    while (r >= y) { q += 1.0; r = fma(-q, y, av); }
    return copysign(r, v);
}

// FSK phase corrections (pyx:121-137): prev = float32(fmod(prev + 2 pi (f_prev - f) t, 2 pi)) at every symbol whose frequency
// differs from its predecessor's — a float32-rounded serial recurrence per message.  One WARP per message: 32 symbols are loaded
// and their increments computed in parallel; only the rounding chain runs in order, from registers, over the symbols that change.
__global__ void __launch_bounds__(128) k_fsk_corrections(const uint8_t* __restrict__ bits, const int64_t* __restrict__ bit_off,
                                                        const int64_t* __restrict__ sym_off, int nmsg, const __grid_constant__ ModParams P,
                                                        float* __restrict__ corr) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double two_pi = 2.0 * M_PI;
    for (int64_t m = warp; m < nmsg; m += nwarps) {
        const uint8_t* b = bits + bit_off[m];
        const int64_t nsym = (bit_off[m + 1] - bit_off[m]) / P.bps;
        float* c = corr + sym_off[m];
        if (nsym <= 0) continue;
        float prev = 0.0f;
        if (lane == 0) c[0] = 0.0f;
        uint32_t carry_idx = symbol_index(b, 0, P.bps);
        for (int64_t base = 1; base < nsym; base += 32) {
            const int64_t s = base + lane;
            const bool valid = s < nsym;
            const uint32_t idx = valid ? symbol_index(b, s, P.bps) : 0u;
            uint32_t pidx = __shfl_up_sync(0xffffffffu, idx, 1);
            if (lane == 0) pidx = carry_idx;
            const int count = (int)min((int64_t)32, nsym - base);
            carry_idx = __shfl_sync(0xffffffffu, idx, count - 1);
            const float f = P.params[idx], fp = P.params[pidx];
            const bool changed = valid && f != fp;
            double term = 0.0;
            if (changed) {
                const float t = __fdiv_rn(__ll2float_rn((long long)(s * (int64_t)P.sps + (int64_t)P.start - 1)), P.sample_rate);
                term = __dmul_rn(__dmul_rn(two_pi, (double)__fsub_rn(fp, f)), (double)t);
            }
            unsigned mask = __ballot_sync(0xffffffffu, changed);
            float mine = prev;
            while (mask) {
                const int l = __ffs(mask) - 1;
                mask &= mask - 1;
                const double tl = __shfl_sync(0xffffffffu, term, l);
                prev = (float)urh_fmod_2pi(__dadd_rn((double)prev, tl));
                if (lane >= l) mine = prev;
            }
            if (valid) c[s] = mine;
        }
    }
}

// GFSK: Gaussian-filtered per-sample frequencies ('same' convolution of the piecewise-constant symbol frequencies).
// The frequency is constant over a symbol, so c[t] = sum_j freq[t-j] g[j] collapses to one term per symbol the window
// touches: f_sym * (G[hi] - G[lo]) with G the running sum of the taps (double) — ~3 terms instead of 2*sps+1.
__global__ void k_gfsk_freqs(const uint8_t* __restrict__ bits, const int64_t* __restrict__ bit_off,
                             const int64_t* __restrict__ smp_off, int nmsg, const __grid_constant__ ModParams P,
                             const double* __restrict__ gsum /* glen+1 prefix sums */, int glen, float* __restrict__ fp_table) {
    // sample indices inside one message fit 32 bits (the host checks): no 64-bit divisions in the per-sample loop
    const int stride = (int)(gridDim.x * blockDim.x);
    for (int m = blockIdx.y; m < nmsg; m += gridDim.y) {   // grid.y is capped at 65535
    const uint8_t* b = bits + bit_off[m];
    const int nsym = (int)((bit_off[m + 1] - bit_off[m]) / P.bps);
    const int nval = nsym * (int)P.sps;
    float* out = fp_table + 2 * smp_off[m];
    for (int k = (int)(blockIdx.x * blockDim.x + threadIdx.x); k < nval; k += stride) {
        // np.convolve(longer, shorter, 'same'): centred on the longer operand
        const int t = (nval >= glen) ? k + (glen - 1) / 2 : k + (nval - 1) / 2;
        // c[t] = sum over i in [max(0, t-glen+1), min(nval-1, t)] of freq[i] * g[t-i]
        int ilo = t - (glen - 1), ihi = t;
        if (ilo < 0) ilo = 0;
        if (ihi > nval - 1) ihi = nval - 1;
        double acc = 0.0;
        for (int i = ilo; i <= ihi;) {
            const int sidx = (int)((unsigned)i / P.sps);
            int iend = (sidx + 1) * (int)P.sps - 1;  // last sample of this symbol
            if (iend > ihi) iend = ihi;
            // taps j = t - i for i in [i, iend]  ->  j in [t - iend, t - i]
            const double w = gsum[t - i + 1] - gsum[t - iend];
            acc += (double)P.params[symbol_index(b, sidx, P.bps)] * w;
            i = iend + 1;
        }
        out[2 * k] = (float)acc;
    }
    }
}

__device__ unsigned long long g_gfsk_blocks[2];   // diagnostics: phase steps taken through an integer prefix sum / one by one

// GFSK phase recurrence (pyx:220-224): phases[i+1] = float32(2*pi*t[i]*(f[i] - f[i+1]) + phases[i]) is a sequential
// float32 accumulation: one WARP per message computes the 32 increments of a block in parallel (coalesced reads) and folds
// them as an integer prefix sum in units of the phase's ulp whenever that is provably the same thing (see FAST BLOCK);
// otherwise in order from registers, exactly as the C loop does.
__global__ void __launch_bounds__(128) k_gfsk_phases(const int64_t* __restrict__ bit_off, const int64_t* __restrict__ smp_off, int nmsg,
                                                    const __grid_constant__ ModParams P, float* __restrict__ fp_table) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double two_pi = 2.0 * M_PI;
    // t = np.arange(start, start + nval, dtype=float32) / sample_rate.  numpy fills a float32 arange as t_i = fl(t0 + fl(fl(i) * d))
    // with t0 = fl(start), d = fl(fl(start + 1) - t0) — not fl(start + i): the two part at i = 2^24 + 1 for start = 1, and from
    // start = 2^31 + 1 on d = 0 (a constant time base).
    const float t0 = __ll2float_rn((long long)P.start);
    const float dt = __fsub_rn(__ll2float_rn((long long)P.start + 1), t0);
    for (int64_t m = warp; m < nmsg; m += nwarps) {
        const int64_t nsym = (bit_off[m + 1] - bit_off[m]) / P.bps;
        const int64_t nval = nsym * P.sps;
        if (nval <= 0) continue;
        float* tab = fp_table + 2 * smp_off[m];
        float ph = P.phi;
        if (lane == 0) tab[1] = ph;
        unsigned long long n_prefix = 0ull, n_serial = 0ull;
        for (int64_t base = 0; base + 1 < nval; base += 32) {
            const int64_t i = base + lane;
            const bool valid = i + 1 < nval;
            double c = 0.0;
            if (valid) {
                const float fcur = tab[2 * i], fnext = tab[2 * (i + 1)];
                const float t = __fdiv_rn(__fadd_rn(t0, __fmul_rn(__ll2float_rn((long long)i), dt)), P.sample_rate);
                c = __dmul_rn(__dmul_rn(two_pi, (double)t), (double)__fsub_rn(fcur, fnext));
            }
            const int count = (int)min((int64_t)32, nval - 1 - base);
            float mine = 0.0f;
            // PREFIX-SUM BLOCK: while the phase stays inside one float binade and sign, float32(c + ph) = ph + round(c / ulp) * ulp, so
            // the recurrence is an INTEGER prefix sum of the quantised increments.  Conditions for the whole 32-step block (else the
            // in-order fold below, exactly as the C loop does):
            //  * ph normal; every partial sum strictly inside the binade [2^23 + 1, 2^24 - 1] ulps, same sign;
            //  * no increment within 1e-6 ulp of a rounding tie (the double addition's own rounding moves the sum by < 2^-29 ulp,
            //    which then cannot change the float rounding).
            // (Consuming a block in segments split at the binade crossings sends more steps through prefix sums, but the longer
            // dependent chain per block makes the kernel slower.)
            bool fast = false;
            {
                const uint32_t pb = __float_as_uint(ph);
                const int e = (int)((pb >> 23) & 0xffu);
                if (e > 0 && e < 255) {
                    const double u = __longlong_as_double((long long)(e - 150 + 1023) << 52);       // ulp of ph's binade = 2^(e-150)
                    const double inv_u = __longlong_as_double((long long)(150 - e + 1023) << 52);
                    const long long m0 = (long long)((pb & 0x7fffffu) | 0x800000u) * ((pb >> 31) ? -1ll : 1ll);
                    const double q = __dmul_rn(c, inv_u);   // exact: a power-of-two scaling
                    const double fr = __dsub_rn(q, floor(q));
                    bool ok = !valid || (fabs(q) < 1.0e12 && fabs(fr - 0.5) > 1.0e-6);
                    const long long k = (valid && ok) ? (long long)rint(q) : 0ll;
                    long long pre = k;   // inclusive prefix over the lanes
#pragma unroll
                    for (int off = 1; off < 32; off <<= 1) {
                        const long long o = __shfl_up_sync(0xffffffffu, pre, off);
                        if (lane >= off) pre += o;
                    }
                    const long long mi = m0 + pre;
                    const long long am = mi < 0 ? -mi : mi;
                    ok = ok && (!valid || (am >= (1ll << 23) + 1 && am <= (1ll << 24) - 1 && ((mi < 0) == (m0 < 0))));
                    fast = __all_sync(0xffffffffu, ok);
                    if (fast) {
                        mine = (float)__dmul_rn((double)mi, u);   // exact: |mi| < 2^24
                        ph = __shfl_sync(0xffffffffu, mine, count - 1);
                        n_prefix += count;
                    }
                }
            }
            if (!fast) {
                for (int l = 0; l < count; l++) {
                    const double cl = __shfl_sync(0xffffffffu, c, l);
                    ph = (float)__dadd_rn(cl, (double)ph);
                    if (lane == l) mine = ph;
                }
                n_serial += count;
            }
            if (valid) tab[2 * (i + 1) + 1] = mine;
        }
        if (lane == 0) {
            atomicAdd(&g_gfsk_blocks[0], n_prefix);
            atomicAdd(&g_gfsk_blocks[1], n_serial);
        }
    }
}

template <typename OUT>
__device__ __forceinline__ OUT mod_cast(float v);
template <> __device__ __forceinline__ float mod_cast<float>(float v) { return v; }
template <> __device__ __forceinline__ int8_t mod_cast<int8_t>(float v) { return (int8_t)(int)v; }
template <> __device__ __forceinline__ int16_t mod_cast<int16_t>(float v) { return (int16_t)(int)v; }

template <typename OUT> struct ModPack;   // two (I, Q) samples as one store
template <> struct ModPack<float> { typedef float4 type; static __device__ __forceinline__ float4 make(float a, float b, float c, float d) { return make_float4(a, b, c, d); } };
template <> struct ModPack<int16_t> { typedef short4 type; static __device__ __forceinline__ short4 make(int16_t a, int16_t b, int16_t c, int16_t d) { return make_short4(a, b, c, d); } };
template <> struct ModPack<int8_t> { typedef char4 type; static __device__ __forceinline__ char4 make(int8_t a, int8_t b, int8_t c, int8_t d) { return make_char4(a, b, c, d); } };

// One modulated sample i (< nval) of message m (pyx:139-172).
template <typename OUT>
__device__ __forceinline__ void mod_sample(int i, int nval, const uint8_t* __restrict__ b, const ModParams& P, const float* __restrict__ corr_m,
                                           const float* __restrict__ fp_m, OUT& outI, OUT& outQ) {
    const double two_pi = 2.0 * M_PI;
    const int s = (int)((unsigned)i / P.sps);
    const uint32_t idx = symbol_index(b, s, P.bps);
    float a = P.a, f = P.f, phi = P.phi, pc = 0.0f;
    if (P.mod_type == URH_MOD_ASK) {
        a = P.params[idx];
        if (a == 0.0f) { outI = (OUT)0; outQ = (OUT)0; return; }   // output stays zero (pyx:148-150)
    } else if (P.mod_type == URH_MOD_FSK) {
        f = P.params[idx];
        pc = corr_m[s];
    } else if (P.mod_type == URH_MOD_PSK || P.mod_type == URH_MOD_OQPSK) {
        phi = P.params[idx];
    } else if (P.mod_type == URH_MOD_GFSK) {
        const float2 fp = *((const float2*)fp_m + i);
        f = fp.x;
        phi = fp.y;
    }
    const float t = __fdiv_rn(__ll2float_rn((long long)i + (long long)P.start), P.sample_rate);
    // current_arg = ((((2.0*M_PI)*f)*t) + phi) + phase_correction, double arithmetic, stored as float
    const double argd = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(two_pi, (double)f), (double)t), (double)phi), (double)pc);
    const float arg = (float)argd;
    float sn, cs;
    int ok;
    urh_glibc_sincosf(arg, &sn, &cs, &ok);
    if (!ok) { sn = sinf(arg); cs = cosf(arg); }
    float I = __fmul_rn(a, cs), Q = __fmul_rn(a, sn);
    if (P.mod_type == URH_MOD_OQPSK) {
        // pyx:168-172: Q of the first symbol and I of the last symbol are zeroed
        if (i < (int)P.sps) Q = 0.0f;
        if (i >= nval - (int)P.sps) I = 0.0f;
    }
    outI = mod_cast<OUT>(I);
    outQ = mod_cast<OUT>(Q);
}

// Every output sample of every message, pause included (zeros): the output is written exactly once (no memset pass before).
// A thread owns the sample pair (2j, 2j + 1) of its message and stores it as one vector when the address allows.
template <typename OUT>
__global__ void __launch_bounds__(256) k_modulate(const uint8_t* __restrict__ bits, const int64_t* __restrict__ bit_off,
                                                 const int64_t* __restrict__ sym_off, const int64_t* __restrict__ smp_off,
                                                 const int64_t* __restrict__ out_off, int nmsg, const __grid_constant__ ModParams P,
                                                 const float* __restrict__ corr, const float* __restrict__ fp_table, OUT* __restrict__ out) {
    typedef typename ModPack<OUT>::type V;
    const int stride = (int)(gridDim.x * blockDim.x);
    for (int m = blockIdx.y; m < nmsg; m += gridDim.y) {   // grid.y is capped at 65535
        const uint8_t* b = bits + bit_off[m];
        const int nsym = (int)((bit_off[m + 1] - bit_off[m]) / P.bps);
        const int nval = nsym * (int)P.sps;
        const int total = (int)(out_off[m + 1] - out_off[m]);   // nval + pause
        OUT* o = out + 2 * out_off[m];
        const float* corr_m = corr ? corr + sym_off[m] : nullptr;
        const float* fp_m = fp_table ? fp_table + 2 * smp_off[m] : nullptr;
        const bool vec_ok = (((uintptr_t)o) % sizeof(V)) == 0;
        const int pairs = (total + 1) >> 1;
        for (int j = (int)(blockIdx.x * blockDim.x + threadIdx.x); j < pairs; j += stride) {
            const int i0 = 2 * j, i1 = 2 * j + 1;
            OUT I0 = (OUT)0, Q0 = (OUT)0, I1 = (OUT)0, Q1 = (OUT)0;
            if (i0 < nval) mod_sample<OUT>(i0, nval, b, P, corr_m, fp_m, I0, Q0);
            if (i1 < nval) mod_sample<OUT>(i1, nval, b, P, corr_m, fp_m, I1, Q1);
            if (vec_ok && i1 < total) {
                *((V*)(o + 2 * (int64_t)i0)) = ModPack<OUT>::make(I0, Q0, I1, Q1);
            } else {
                o[2 * (int64_t)i0] = I0;
                o[2 * (int64_t)i0 + 1] = Q0;
                if (i1 < total) {
                    o[2 * (int64_t)i1] = I1;
                    o[2 * (int64_t)i1 + 1] = Q1;
                }
            }
        }
    }
}

// GFSK (frequency, phase) table of a batch: per-sample filtered frequencies, then the phase recurrence.  fp_table holds
// 2 * smp_off[nmsg] floats; max_samples is the longest message in samples.
static int gfsk_table(urh_ctx* ctx, const uint8_t* d_bits, const int64_t* d_bit_off, const int64_t* d_smp_off, int nmsg, const ModParams& P,
                      int64_t max_samples, const float* h_gauss_fir, int gauss_len, float* fp_table) {
    if (!h_gauss_fir || gauss_len <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "GFSK needs the gaussian filter taps");
    std::vector<double> gsum((size_t)gauss_len + 1, 0.0);
    for (int j = 0; j < gauss_len; j++) gsum[j + 1] = gsum[j] + (double)h_gauss_fir[j];
    double* d_gsum;
    URH_CHECK(urh_arena(ctx, (size_t)gauss_len + 1, &d_gsum));
    URH_CUDA(ctx, cudaMemcpyAsync(d_gsum, gsum.data(), (gauss_len + 1) * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const unsigned gx = (unsigned)max((int64_t)1, min(urh_div_up(max_samples, 256), (int64_t)ctx->sm_count * 8));
    const dim3 grid(gx, (unsigned)min(nmsg, 65535));
    URH_LAUNCH(ctx, k_gfsk_freqs, grid, 256, 0, d_bits, d_bit_off, d_smp_off, nmsg, P, d_gsum, gauss_len, fp_table);
    URH_LAUNCH(ctx, k_gfsk_phases, (unsigned)min((int64_t)urh_div_up(nmsg, 4), (int64_t)ctx->sm_count * 16), 128, 0, d_bit_off, d_smp_off, nmsg, P,
               fp_table);
    return URH_OK;
}

// Batch modulate.  d_bits: concatenated bit arrays (uint8, already OQPSK-shuffled if needed);
// h_bit_off[nmsg+1]: bit offsets; h_out_off[nmsg+1]: output SAMPLE offsets (message m occupies
// [h_out_off[m], h_out_off[m+1]) = symbols*sps + pause samples); d_out is zero-filled here.
extern "C" int urh_modulate_batch(urh_ctx* ctx, const uint8_t* d_bits, const int64_t* h_bit_off, const int64_t* h_out_off,
                                  int nmsg, uint32_t samples_per_symbol, int mod_type, const float* h_params, int nparams,
                                  int bits_per_symbol, float carrier_amplitude, float carrier_frequency, float carrier_phase,
                                  float sample_rate, uint32_t start, int out_dtype, const float* h_gauss_fir, int gauss_len,
                                  void* d_out) {
    if (nmsg <= 0) return URH_OK;
    if (mod_type != URH_MOD_ASK && mod_type != URH_MOD_FSK && mod_type != URH_MOD_PSK && mod_type != URH_MOD_GFSK &&
        mod_type != URH_MOD_OQPSK)
        URH_FAIL(ctx, URH_ERR_MODULATION, "unknown modulation type");
    if (mod_type == URH_MOD_OQPSK && bits_per_symbol != 2) URH_FAIL(ctx, URH_ERR_MODULATION, "OQPSK needs bits_per_symbol == 2");
    if (out_dtype != URH_DT_I8 && out_dtype != URH_DT_I16 && out_dtype != URH_DT_F32)
        URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype for modulation");
    if (bits_per_symbol < 1 || bits_per_symbol > 8 || nparams > 256 || nparams < (1 << bits_per_symbol))
        URH_FAIL(ctx, URH_ERR_INVALID, "bits_per_symbol / parameters mismatch");
    urh_arena_reset(ctx);
    ModParams P;
    memset(&P, 0, sizeof(P));
    P.sps = samples_per_symbol; P.mod_type = mod_type; P.bps = bits_per_symbol; P.a = carrier_amplitude;
    P.f = carrier_frequency; P.phi = carrier_phase; P.sample_rate = sample_rate; P.start = start; P.out_dtype = out_dtype;
    P.nparams = nparams;
    memcpy(P.params, h_params, sizeof(float) * nparams);
    // per-message offsets: symbols and modulated (non-pause) samples
    std::vector<int64_t> sym_off(nmsg + 1, 0), smp_off(nmsg + 1, 0);
    int64_t max_samples = 0, max_total = 0;
    for (int m = 0; m < nmsg; m++) {
        const int64_t nsym = (h_bit_off[m + 1] - h_bit_off[m]) / bits_per_symbol;
        sym_off[m + 1] = sym_off[m] + nsym;
        smp_off[m + 1] = smp_off[m] + nsym * samples_per_symbol;
        if (nsym * (int64_t)samples_per_symbol > max_samples) max_samples = nsym * samples_per_symbol;
        if (h_out_off[m + 1] - h_out_off[m] < nsym * (int64_t)samples_per_symbol) URH_FAIL(ctx, URH_ERR_INVALID, "output offsets too small");
        if (h_out_off[m + 1] - h_out_off[m] >= ((int64_t)1 << 31) - 2)
            URH_FAIL(ctx, URH_ERR_INVALID, "one message of >= 2^31 samples: split it (the float32 time base of the reference is exhausted at 2^24)");
        if (h_out_off[m + 1] - h_out_off[m] > max_total) max_total = h_out_off[m + 1] - h_out_off[m];
    }
    int64_t *d_bit_off, *d_sym_off, *d_smp_off, *d_out_off;
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_bit_off));
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_sym_off));
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_smp_off));
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_out_off));
    const size_t ob = (size_t)(nmsg + 1) * sizeof(int64_t);
    URH_CUDA(ctx, cudaMemcpyAsync(d_bit_off, h_bit_off, ob, cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(d_sym_off, sym_off.data(), ob, cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(d_smp_off, smp_off.data(), ob, cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(d_out_off, h_out_off, ob, cudaMemcpyHostToDevice, ctx->stream));
    // the modulation kernel writes every output sample once, pauses included: no memset pass over the (write-only) output
    float *corr = nullptr, *fp_table = nullptr;
    if (mod_type == URH_MOD_FSK) {
        URH_CHECK(urh_arena(ctx, (size_t)sym_off[nmsg] + 1, &corr));
        URH_LAUNCH(ctx, k_fsk_corrections, (unsigned)min((int64_t)urh_div_up(nmsg, 4), (int64_t)ctx->sm_count * 16), 128, 0, d_bits, d_bit_off, d_sym_off, nmsg, P, corr);
    }
    if (mod_type == URH_MOD_GFSK) {
        URH_CHECK(urh_arena(ctx, (size_t)smp_off[nmsg] * 2 + 2, &fp_table));
        URH_CHECK(gfsk_table(ctx, d_bits, d_bit_off, d_smp_off, nmsg, P, max_samples, h_gauss_fir, gauss_len, fp_table));
    }
    const unsigned gp = (unsigned)max((int64_t)1, min(urh_div_up(urh_div_up(max_total, 2), 256), (int64_t)ctx->sm_count * 8));
    const dim3 gridp(gp, (unsigned)min(nmsg, 65535));
    if (out_dtype == URH_DT_F32)
        URH_LAUNCH(ctx, k_modulate<float>, gridp, 256, 0, d_bits, d_bit_off, d_sym_off, d_smp_off, d_out_off, nmsg, P, corr, fp_table, (float*)d_out);
    else if (out_dtype == URH_DT_I16)
        URH_LAUNCH(ctx, k_modulate<int16_t>, gridp, 256, 0, d_bits, d_bit_off, d_sym_off, d_smp_off, d_out_off, nmsg, P, corr, fp_table, (int16_t*)d_out);
    else
        URH_LAUNCH(ctx, k_modulate<int8_t>, gridp, 256, 0, d_bits, d_bit_off, d_sym_off, d_smp_off, d_out_off, nmsg, P, corr, fp_table, (int8_t*)d_out);
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the offset vectors above are host temporaries
    return URH_OK;
}

// diagnostics of the GFSK phase kernel since the last call: {phase steps taken through an integer prefix sum, steps taken one by one}
extern "C" int urh_modulate_stats(urh_ctx* ctx, int64_t* h_out2) {
    unsigned long long v[2] = {0ull, 0ull};
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    URH_CUDA(ctx, cudaMemcpyFromSymbol(v, g_gfsk_blocks, sizeof(v)));
    const unsigned long long z[2] = {0ull, 0ull};
    URH_CUDA(ctx, cudaMemcpyToSymbol(g_gfsk_blocks, z, sizeof(z)));
    h_out2[0] = (int64_t)v[0];
    h_out2[1] = (int64_t)v[1];
    return URH_OK;
}

// Test entry point: only the GFSK table of a batch (k_gfsk_freqs + k_gfsk_phases, as urh_modulate_batch runs them) into
// d_table = (sum of symbols * sps, 2) float32 (frequency, phase) rows, message after message.
extern "C" int urh_modulate_gfsk_table(urh_ctx* ctx, const uint8_t* d_bits, const int64_t* h_bit_off, int nmsg, uint32_t samples_per_symbol,
                                       const float* h_params, int nparams, int bits_per_symbol, float carrier_phase, float sample_rate,
                                       uint32_t start, const float* h_gauss_fir, int gauss_len, float* d_table) {
    if (nmsg <= 0) return URH_OK;
    if (bits_per_symbol < 1 || bits_per_symbol > 8 || nparams > 256 || nparams < (1 << bits_per_symbol))
        URH_FAIL(ctx, URH_ERR_INVALID, "bits_per_symbol / parameters mismatch");
    urh_arena_reset(ctx);
    ModParams P;
    memset(&P, 0, sizeof(P));
    P.sps = samples_per_symbol; P.mod_type = URH_MOD_GFSK; P.bps = bits_per_symbol; P.phi = carrier_phase; P.sample_rate = sample_rate;
    P.start = start; P.nparams = nparams;
    memcpy(P.params, h_params, sizeof(float) * nparams);
    std::vector<int64_t> smp_off(nmsg + 1, 0);
    int64_t max_samples = 0;
    for (int m = 0; m < nmsg; m++) {
        const int64_t nval = (h_bit_off[m + 1] - h_bit_off[m]) / bits_per_symbol * samples_per_symbol;
        if (nval >= ((int64_t)1 << 31) - 2) URH_FAIL(ctx, URH_ERR_INVALID, "one message of >= 2^31 samples: split it");
        smp_off[m + 1] = smp_off[m] + nval;
        if (nval > max_samples) max_samples = nval;
    }
    int64_t *d_bit_off, *d_smp_off;
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_bit_off));
    URH_CHECK(urh_arena(ctx, (size_t)nmsg + 1, &d_smp_off));
    const size_t ob = (size_t)(nmsg + 1) * sizeof(int64_t);
    URH_CUDA(ctx, cudaMemcpyAsync(d_bit_off, h_bit_off, ob, cudaMemcpyHostToDevice, ctx->stream));
    URH_CUDA(ctx, cudaMemcpyAsync(d_smp_off, smp_off.data(), ob, cudaMemcpyHostToDevice, ctx->stream));
    URH_CHECK(gfsk_table(ctx, d_bits, d_bit_off, d_smp_off, nmsg, P, max_samples, h_gauss_fir, gauss_len, d_table));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the offset vectors above are host temporaries
    return URH_OK;
}

// Test entry point: the modulator's device math on device arrays — urh_glibc_sincosf(x[i]) -> sn[i], cs[i], ok[i] and
// urh_fmod_2pi(v[j]) -> r[j] — for comparison with libm's sinf / cosf / fmod.
__global__ void k_selftest_modmath(const float* __restrict__ x, int64_t n, float* __restrict__ sn, float* __restrict__ cs, int* __restrict__ ok,
                                   const double* __restrict__ v, int64_t nv, double* __restrict__ r) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float s, c;
        int o;
        urh_glibc_sincosf(x[i], &s, &c, &o);
        sn[i] = s;
        cs[i] = c;
        ok[i] = o;
    }
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nv; j += stride) r[j] = urh_fmod_2pi(v[j]);
}

extern "C" int urh_selftest_modmath(urh_ctx* ctx, const float* d_x, int64_t n, float* d_sn, float* d_cs, int* d_ok, const double* d_v,
                                    int64_t nv, double* d_r) {
    if (n <= 0 && nv <= 0) return URH_OK;
    const unsigned g = (unsigned)max((int64_t)1, min(urh_div_up(max(n, nv), 256), (int64_t)ctx->sm_count * 8));
    URH_LAUNCH(ctx, k_selftest_modmath, g, 256, 0, d_x, n, d_sn, d_cs, d_ok, d_v, nv, d_r);
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return URH_OK;
}
