/*
 * urh_oracle.c — CPU restatement (plain C) of the reference's DSP kernels for the IQ hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (urh_b200/) may import, link or call this file;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, and
 * only as the checker / the timed CPU baseline.
 *
 * Parity is PINNED: tests/test_oracle.py checks every function here bit-for-bit against the reference's
 * own compiled Cython kernels (oracle/_ref, built by oracle/build_ref.py from /root/reference) and
 * against the golden vectors under tests/golden/ generated from the unmodified reference.
 *
 * Each function cites the reference lines it restates (paths relative to the reference root).
 * Build: gcc -O2 -fopenmp -ffp-contract=off -shared -fPIC (oracle/Makefile).  libm's float routines
 * (atan2f, sqrtf, log10f, cosf, sinf) are the ones the reference binds (C++ overloads on float).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { DT_I8 = 0, DT_U8 = 1, DT_I16 = 2, DT_U16 = 3, DT_F32 = 4 };
enum { MOD_ASK = 0, MOD_FSK = 1, MOD_PSK = 2, MOD_QAM = 3, MOD_GFSK = 4, MOD_OQPSK = 5 };

static inline float iq_at(const void* iq, int dtype, int64_t idx) {
    switch (dtype) {
        case DT_I8: return (float)((const int8_t*)iq)[idx];
        case DT_U8: return (float)((const uint8_t*)iq)[idx];
        case DT_I16: return (float)((const int16_t*)iq)[idx];
        case DT_U16: return (float)((const uint16_t*)iq)[idx];
        default: return ((const float*)iq)[idx];
    }
}

/* src/urh/cythonext/signal_functions.pyx:31-44 */
float oracle_noise_value(int mod_type) {
    switch (mod_type) {
        case MOD_ASK: return 0.0f;
        case MOD_FSK:
        case MOD_PSK:
        case MOD_OQPSK: return -4.0f;
        case MOD_QAM: return 0.0f * -4.0f;
        default: return 0.0f;
    }
}

/* std::complex<float> product (a+ib)(c+id) as GCC evaluates it without -ffast-math: the naive product, and when both parts
 * are NaN, libgcc's __mulsc3 recovery (C99 Annex G, G.5.1): an infinite operand gives an infinite result */
static inline void cmulf(float a, float b, float c, float d, float* re, float* im) {
    const float ac = a * c, bd = b * d, ad = a * d, bc = b * c;
    *re = ac - bd;
    *im = ad + bc;
    if (isnan(*re) && isnan(*im)) {
        int recalc = 0;
        if (isinf(a) || isinf(b)) {
            a = copysignf(isinf(a) ? 1.0f : 0.0f, a);
            b = copysignf(isinf(b) ? 1.0f : 0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = 1;
        }
        if (isinf(c) || isinf(d)) {
            c = copysignf(isinf(c) ? 1.0f : 0.0f, c);
            d = copysignf(isinf(d) ? 1.0f : 0.0f, d);
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            recalc = 1;
        }
        if (!recalc && (isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc))) {
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = 1;
        }
        if (recalc) {
            *re = INFINITY * (a * c - b * d);
            *im = INFINITY * (a * d + b * c);
        }
    }
}

/* Costas loop — src/urh/cythonext/signal_functions.pyx:252-330 */
static void costas_from(const void* iq, int dtype, int64_t n, float noise_sqrd, int loop_order, float bandwidth, float* out,
                        int64_t first, float freq0, float phase0, float* end_state);
static void costas(const void* iq, int dtype, int64_t n, float noise_sqrd, int loop_order, float bandwidth, float* out) {
    if (n > 0) out[0] = 0.0f; /* np.empty in the reference: undefined; we pin it to 0 */
    costas_from(iq, dtype, n, noise_sqrd, loop_order, bandwidth, out, 1, 0.0f, 1.5f, 0);
}

/* The loop of signal_functions.pyx:289-328 over samples [first, n), starting from the loop state (freq0, phase0); the state
 * after the last sample goes to end_state[0..1].  costas() above is the reference's call (first = 1, state 0 / 1.5); a later start
 * with the state a preceding segment ended in continues that run (test oracle for captures sharded over GPUs). */
static void costas_from(const void* iq, int dtype, int64_t n, float noise_sqrd, int loop_order, float bandwidth, float* out,
                        int64_t first, float freq0, float phase0, float* end_state) {
    const float damping = (float)(sqrt(2.0) / 2.0);
    const double den = (1.0 + ((2.0 * damping) * bandwidth)) + (bandwidth * bandwidth);
    const float alpha = (float)(((double)((4.0 * damping) * bandwidth)) / den);
    const float beta = (float)(((double)((4.0 * bandwidth) * bandwidth)) / den);
    float scale, shift;
    switch (dtype) {
        case DT_I8: scale = 127.5f; shift = 0.5f; break;
        case DT_U8: scale = 127.5f; shift = -127.5f; break;
        case DT_I16: scale = 32767.5f; shift = 0.5f; break;
        case DT_U16: scale = 65535.0f; shift = -32767.5f; break;
        default: scale = 1.0f; shift = 0.0f; break;
    }
    if (loop_order > 4) loop_order = 4;
    float freq = freq0, err = 0.0f, phase = phase0;
    for (int64_t i = first; i < n; i++) {
        const float re = iq_at(iq, dtype, 2 * i), im = iq_at(iq, dtype, 2 * i + 1);
        if (re * re + im * im <= noise_sqrd) {
            out[i] = -4.0f;
            continue;
        }
        const float rf = (re + shift) / scale, jf = (im + shift) / scale;
        /* rf + 1j*jf and cosf(-p) + 1j*sinf(-p): 1j*v = (0*v - 1*0, 0*0 + 1*v) */
        float pr, pi;
        cmulf(0.0f, 1.0f, jf, 0.0f, &pr, &pi);
        const float sr = rf + pr, si = 0.0f + pi;
        cmulf(0.0f, 1.0f, sinf(-phase), 0.0f, &pr, &pi);
        const float nr = cosf(-phase) + pr, ni = 0.0f + pi;
        float xr, xi;
        cmulf(nr, ni, sr, si, &xr, &xi);
        if (loop_order == 2) err = xi * xr;
        else if (loop_order == 4) {
            const float f1 = xr > 0.0 ? 1.0f : -1.0f, f2 = xi > 0.0 ? 1.0f : -1.0f;
            err = f1 * xi - f2 * xr;
        }
        err = err < -1.0f ? -1.0f : (err > 1.0f ? 1.0f : err);
        freq = freq + beta * err;
        phase = phase + (freq + alpha * err);
        while (phase > (2.0 * M_PI)) phase = (float)(phase - (2.0 * M_PI));
        while (phase < (-2.0 * M_PI)) phase = (float)(phase + (2.0 * M_PI));
        freq = freq < -1.0f ? -1.0f : (freq > 1.0f ? 1.0f : freq);
        if (loop_order == 2) out[i] = xr;
        else if (loop_order == 4) out[i] = (float)((2.0 * xr) + xi);
    }
    if (end_state) { end_state[0] = freq; end_state[1] = phase; }
}

/* test hook: continue a Costas run from a known loop state (see costas_from) */
int oracle_costas_from(const void* iq, int dtype, int64_t n, float noise_mag, int loop_order, float bandwidth, float freq0, float phase0,
                       float* out, float* end_state) {
    const float noise_sqrd = noise_mag * noise_mag;
    costas_from(iq, dtype, n, noise_sqrd, loop_order, bandwidth, out, 0, freq0, phase0, end_state);
    return 0;
}

/* afp_demod — src/urh/cythonext/signal_functions.pyx:333-378 */
int oracle_afp_demod(const void* iq, int dtype, int64_t n, float noise_mag, int mod_type, int mod_order,
                     float costas_bw, float* out) {
    if (n <= 2) {
        memset(out, 0, (size_t)(n > 0 ? n : 0) * sizeof(float));
        return 0;
    }
    const float NOISE = oracle_noise_value(mod_type);
    const float noise_sqrd = noise_mag * noise_mag;
    float max_mag;
    switch (dtype) {
        case DT_I8: max_mag = (float)sqrt(32513.0); break;
        case DT_U8: max_mag = (float)sqrt(65025.0); break;
        case DT_I16: max_mag = (float)sqrt(2147418113.0); break;
        case DT_U16: max_mag = (float)sqrt(4294836225.0); break;
        case DT_F32: max_mag = (float)sqrt(2.0); break;
        default: return -3;
    }
    if (mod_type == MOD_PSK) {
        costas(iq, dtype, n, noise_sqrd, mod_order, costas_bw, out);
        return 0;
    }
    memset(out, 0, (size_t)n * sizeof(float));
    out[0] = NOISE;
    int64_t i;
#pragma omp parallel for schedule(static)
    for (i = 1; i < n; i++) {
        const float re = iq_at(iq, dtype, 2 * i), im = iq_at(iq, dtype, 2 * i + 1);
        const float mag = re * re + im * im;
        if (mag <= noise_sqrd) {
            out[i] = NOISE;
            continue;
        }
        if (mod_type == MOD_ASK) {
            out[i] = (float)(sqrtf(mag) / ((double)max_mag));
        } else if (mod_type == MOD_FSK) {
            const float a = iq_at(iq, dtype, 2 * (i - 1)), b = iq_at(iq, dtype, 2 * (i - 1) + 1);
            float tr, ti, ur, ui, xr, xi;
            cmulf(0.0f, 1.0f, b, 0.0f, &tr, &ti);   /* 1j * x[i-1].imag */
            const float A = a - tr, B = 0.0f - ti;  /* x[i-1].real - (...) */
            cmulf(0.0f, 1.0f, im, 0.0f, &ur, &ui);  /* 1j * imag */
            const float Cc = re + ur, D = 0.0f + ui;
            cmulf(A, B, Cc, D, &xr, &xi);
            out[i] = atan2f(xi, xr);
        }
    }
    return 0;
}

/* get_center_thresholds — src/urh/cythonext/signal_functions.pyx:380-390 */
void oracle_center_thresholds(float center, float spacing, int order, float* out) {
    const int n = order / 2;
    for (int i = 0; i < n; i++) out[i] = center - (n - (i + 1)) * spacing;
    for (int i = n; i < order - 1; i++) out[i] = center + (i + 1 - n) * spacing;
}

/* grab_pulse_lens — src/urh/cythonext/signal_functions.pyx:392-495.
 * out_rows must hold (n,2) int64; returns the number of rows. */
int64_t oracle_grab_pulse_lens(const float* samples, int64_t n, float center, uint16_t tolerance, int mod_type,
                               uint32_t samples_per_symbol, uint8_t bits_per_symbol, float center_spacing,
                               int64_t* out_rows) {
    if (n == 0) return 0;
    const int is_ask = mod_type == MOD_ASK;
    const float NOISE = oracle_noise_value(mod_type);
    const int order = 1 << bits_per_symbol;
    float* thr = (float*)malloc(sizeof(float) * (size_t)(order > 1 ? order - 1 : 1));
    int64_t* count = (int64_t*)calloc((size_t)order, sizeof(int64_t));
    oracle_center_thresholds(center, center_spacing, order, thr);
    int64_t rows = 0, pulse = 0, pause_run = 0;
    int cur, fresh;
    float s = 0.0f;
    /* initial state: PAUSE if samples[0] is the noise sentinel, else the class of the literal 0.0 (pyx:421-429) */
    if (samples[0] == NOISE) cur = -1;
    else {
        cur = order - 1;
        for (int k = 0; k < order - 1; k++)
            if (s <= thr[k]) { cur = k; break; }
    }
    for (int64_t i = 0; i < n; i++) {
        pulse++;
        s = samples[i];
        if (s == NOISE) fresh = -1;
        else {
            fresh = order - 1;
            for (int k = 0; k < order - 1; k++)
                if (s <= thr[k]) { fresh = k; break; }
        }
        pause_run = (fresh == -1) ? pause_run + 1 : 0;
        for (int j = 0; j < order; j++) count[j] = (j == fresh) ? count[j] + 1 : 0;
        if (cur == fresh) continue;
        int next = -42;
        if (pause_run > tolerance) next = -1;
        else
            for (int j = 0; j < order; j++)
                if (count[j] > tolerance) { next = j; break; }
        if (next == -42) continue;
        if (is_ask && cur == -1 && (pulse - tolerance) < (int64_t)samples_per_symbol) cur = 0;
        if (rows > 0 && out_rows[2 * (rows - 1)] == cur) out_rows[2 * (rows - 1) + 1] += pulse - tolerance;
        else {
            out_rows[2 * rows] = cur;
            out_rows[2 * rows + 1] = pulse - tolerance;
            rows++;
        }
        pulse = tolerance;
        cur = next;
    }
    if (rows < n) {
        if (rows > 0 && out_rows[2 * (rows - 1)] == cur) out_rows[2 * (rows - 1) + 1] += pulse - tolerance;
        else {
            out_rows[2 * rows] = cur;
            out_rows[2 * rows + 1] = pulse - tolerance;
            rows++;
        }
    }
    free(thr);
    free(count);
    return rows;
}

/* get_magnitudes — src/urh/cythonext/util.pyx:128-136 (float: sqrtf of a float sum; ints: int arithmetic, double sqrt) */
void oracle_get_magnitudes(const void* iq, int dtype, int64_t n, double* out) {
    for (int64_t i = 0; i < n; i++) {
        if (dtype == DT_F32) {
            const float re = ((const float*)iq)[2 * i], im = ((const float*)iq)[2 * i + 1];
            out[i] = (double)sqrtf(re * re + im * im);
        } else {
            int32_t re, im;
            switch (dtype) {
                case DT_I8: re = ((const int8_t*)iq)[2 * i]; im = ((const int8_t*)iq)[2 * i + 1]; break;
                case DT_U8: re = ((const uint8_t*)iq)[2 * i]; im = ((const uint8_t*)iq)[2 * i + 1]; break;
                case DT_I16: re = ((const int16_t*)iq)[2 * i]; im = ((const int16_t*)iq)[2 * i + 1]; break;
                default: re = ((const uint16_t*)iq)[2 * i]; im = ((const uint16_t*)iq)[2 * i + 1]; break;
            }
            /* C int arithmetic (wraps for large uint16 values exactly like the reference's UB does in practice) */
            const int32_t ssum = (int32_t)((uint32_t)re * (uint32_t)re + (uint32_t)im * (uint32_t)im);
            out[i] = sqrt((double)ssum);
        }
    }
}

/* segment_messages_from_magnitudes — src/urh/cythonext/auto_interpretation.pyx:55-111.
 * mags float32 or float64 (is_f64).  out pairs (start,end) must hold n/10+2 entries; returns count. */
int64_t oracle_segment_messages(const void* mags, int is_f64, int64_t n, float noise_threshold, int64_t* out) {
    if (n == 0) return 0;
    const unsigned int tol = 10;
    unsigned int above = 0, below = 0;
    uint64_t start = 0;
    int64_t cnt = 0;
#define MAG(i) (is_f64 ? ((const double*)mags)[i] : (double)((const float*)mags)[i])
    int state = (MAG(0) > noise_threshold) ? 1 : -1;
    for (uint64_t i = 0; i < (uint64_t)n; i++) {
        const int is_above = MAG(i) > noise_threshold;
        if (state == 1) below = is_above ? 0 : below + 1;
        else above = is_above ? above + 1 : 0;
        if (state == 1 && below >= tol) {
            state = -1;
            out[2 * cnt] = (int64_t)start;
            out[2 * cnt + 1] = (int64_t)(i - below);
            cnt++;
            below = above = 0;
        } else if (state == -1 && above >= tol) {
            state = 1;
            start = i - above;
            below = above = 0;
        }
    }
    if (state == 1 && start < (uint64_t)n - below) {
        out[2 * cnt] = (int64_t)start;
        out[2 * cnt + 1] = (int64_t)((uint64_t)n - below);
        cnt++;
    }
#undef MAG
    return cnt;
}

/* fir_filter — src/urh/cythonext/signal_functions.pyx:513-525 (complex64 accumulation order preserved) */
void oracle_fir_filter(const float* x, int64_t n, const float* taps, int64_t m, float* out) {
    float* acc = (float*)calloc((size_t)(n + m) * 2, sizeof(float));
    for (int64_t i = 0; i < n; i++)
        for (int64_t j = 0; j < m; j++) {
            float pr, pi;
            cmulf(x[2 * i], x[2 * i + 1], taps[2 * j], taps[2 * j + 1], &pr, &pi);
            acc[2 * (i + j)] += pr;
            acc[2 * (i + j) + 1] += pi;
        }
    memcpy(out, acc, (size_t)n * 2 * sizeof(float));
    free(acc);
}

/* arr2decibel — src/urh/cythonext/util.pyx:38-48: 10.0f * log10f(re^2 + im^2), all float32 */
void oracle_arr2decibel(const float* x, int64_t count, float* out) {
    for (int64_t i = 0; i < count; i++) {
        const float re = x[2 * i], im = x[2 * i + 1];
        out[i] = 10.0f * log10f(re * re + im * im);
    }
}

/* bit_array_to_number — src/urh/cythonext/util.pyx:50-61 (MSB first) */
static uint64_t bits_to_number(const uint8_t* bits, int64_t end, int64_t start) {
    if (end < 1) return 0;
    uint64_t r = 0, acc = 1;
    for (int64_t i = start; i < end; i++) {
        r += bits[end - 1 - i + start] * acc;
        acc *= 2;
    }
    return r;
}

/* modulate_c / __modulate — src/urh/cythonext/signal_functions.pyx:56-177 (ASK / FSK / PSK / OQPSK; GFSK takes
 * the per-sample frequency/phase table computed by the caller — numpy convolve lives on the Python side).
 * out: (total,2) of out_dtype (DT_I8 / DT_I16 / DT_F32), zero-initialised by the caller.
 * `bits` must already be the OQPSK-shuffled bits when mod_type == OQPSK. */
int oracle_modulate(const uint8_t* bits, int64_t num_bits, uint32_t sps, int mod_type, const float* params,
                    uint16_t bps, float a0, float f0, float phi0, float sample_rate, uint32_t pause, uint32_t start,
                    int out_dtype, const float* gfsk_freq_phase, void* out) {
    const uint32_t total_symbols = (uint32_t)(num_bits / bps);
    const int64_t total_samples = (int64_t)total_symbols * sps + pause;
    if (num_bits == 0) return 0;
    float* corr = NULL;
    if (mod_type == MOD_FSK && total_symbols > 0) {
        corr = (float*)malloc(sizeof(float) * total_symbols);
        corr[0] = 0.0f;
        for (int64_t s = 1; s < total_symbols; s++) {
            const float f = params[bits_to_number(bits, (s + 1) * bps, s * bps)];
            const float fp = params[bits_to_number(bits, s * bps, (s - 1) * bps)];
            if (f != fp) {
                const float t = ((float)((s * sps + start) - 1)) / sample_rate;
                corr[s] = (float)fmod(corr[s - 1] + (((2.0 * M_PI) * (fp - f)) * t), 2.0 * M_PI);
            } else corr[s] = corr[s - 1];
        }
    }
    for (int64_t s = 0; s < total_symbols; s++) {
        const uint64_t idx = bits_to_number(bits, (s + 1) * bps, s * bps);
        float a = a0, f = f0, phi = phi0, pc = 0.0f;
        if (mod_type == MOD_ASK) {
            a = params[idx];
            if (a == 0) continue;
        } else if (mod_type == MOD_FSK) {
            f = params[idx];
            pc = corr[s];
        } else if (mod_type == MOD_PSK || mod_type == MOD_OQPSK) phi = params[idx];
        for (int64_t i = s * sps; i < (s + 1) * (int64_t)sps; i++) {
            const float t = ((float)(i + start)) / sample_rate;
            if (mod_type == MOD_GFSK) {
                f = gfsk_freq_phase[2 * i];
                phi = gfsk_freq_phase[2 * i + 1];
            }
            const float arg = (float)(((((2.0 * M_PI) * f) * t) + phi) + pc);
            const float I = a * cosf(arg), Q = a * sinf(arg);
            if (out_dtype == DT_I8) {
                ((int8_t*)out)[2 * i] = (int8_t)I;
                ((int8_t*)out)[2 * i + 1] = (int8_t)Q;
            } else if (out_dtype == DT_I16) {
                ((int16_t*)out)[2 * i] = (int16_t)I;
                ((int16_t*)out)[2 * i + 1] = (int16_t)Q;
            } else {
                ((float*)out)[2 * i] = I;
                ((float*)out)[2 * i + 1] = Q;
            }
        }
    }
    if (mod_type == MOD_OQPSK) {
        for (int64_t i = 0; i < sps; i++) {
            if (out_dtype == DT_I8) ((int8_t*)out)[2 * i + 1] = 0;
            else if (out_dtype == DT_I16) ((int16_t*)out)[2 * i + 1] = 0;
            else ((float*)out)[2 * i + 1] = 0;
        }
        for (int64_t i = total_samples - pause - sps; i < total_samples - pause; i++) {
            if (out_dtype == DT_I8) ((int8_t*)out)[2 * i] = 0;
            else if (out_dtype == DT_I16) ((int16_t*)out)[2 * i] = 0;
            else ((float*)out)[2 * i] = 0;
        }
    }
    free(corr);
    return 0;
}

/* median_filter — src/urh/cythonext/auto_interpretation.pyx:211-240: window [i, i+k) truncated at the end,
 * float32 buffer, returns buffer[k//2] after sorting */
static int cmp_float(const void* a, const void* b) {
    const float x = *(const float*)a, y = *(const float*)b;
    return (x > y) - (x < y);
}
void oracle_median_filter(const double* data, int64_t n, unsigned int k, float* out) {
    float* buf = (float*)malloc(sizeof(float) * (k ? k : 1));
    for (int64_t i = 0; i < n; i++) {
        unsigned int kk = k;
        if ((uint64_t)i + kk > (uint64_t)n) kk = (unsigned int)(n - i);
        for (unsigned int j = 0; j < kk; j++) buf[j] = (float)data[i + j];
        qsort(buf, kk, sizeof(float), cmp_float);
        out[i] = buf[kk / 2];
    }
    free(buf);
}

/* get_plateau_lengths — src/urh/cythonext/auto_interpretation.pyx:179-208.  Returns count; out must hold n. */
int64_t oracle_plateau_lengths(const float* rect, int64_t n, float center, int percentage, uint64_t* out) {
    if (n == 0) return 0;
    int state = rect[0] <= center ? -1 : 1;
    uint64_t plateau = 0, sum = 0;
    int64_t cnt = 0;
    for (uint64_t i = 0; i < (uint64_t)n; i++) {
        if (sum >= (uint64_t)percentage * (uint64_t)n / 100) break;
        const int ns = rect[i] <= center ? -1 : 1;
        if (ns == state) plateau++;
        else {
            out[cnt++] = plateau;
            sum += plateau;
            state = ns;
            plateau = 1;
        }
    }
    return cnt;
}
