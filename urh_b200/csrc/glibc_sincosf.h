// Bit-faithful restatement of glibc 2.39 sinf / cosf for every finite argument: the small / medium ranges the
// Costas loop needs (signal_functions.pyx:301, phase wrapped to +-2*pi) and the large-argument reduction the
// modulator needs (signal_functions.pyx:163-166: 2*pi*f*t reaches 1e5..1e7 rad).
//
// Provenance of every constant and of the operation order: NOT glibc source, but the machine code and
// .rodata of THIS image's /usr/lib/x86_64-linux-gnu/libm.so.6 (glibc 2.39-0ubuntu8.5, build-id
// 0d9969fe206760d250ec30a5a9be18aefbf84ea8), read with objdump/readelf in round 1:
//   * sinf / cosf are IFUNCs; on CPUs with FMA+AVX2 (the x86-64 hosts the GPUs sit in) they resolve
//     to the FMA variants at 0x7e800 / 0x7e330, whose double-precision polynomial steps are contracted
//     into vfmadd exactly as written below (fma() here == one IEEE fused operation, as on the GPU);
//   * the 14-double table __sincosf_table[2] sits at 0xb8120 (signs, 2/pi*2^24, pi/2, c0,c1,s1,c2,s2,c3,s3,c4);
//     entry [1] negates the cosine polynomial.
// The non-FMA (SSE2) variant differs only in the last bit of the double intermediates (observable in the
// float result with probability ~2^-29 per call).  tests/test_sincosf_restatement.py (|x| < 120) and
// tests/test_modulator_pin.py (|x| >= 120) pin this header against libm bit-for-bit on the CPU;
// tests/test_gpu_modulator_exact.py pins the device build over the whole float range.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDA_ARCH__)
#define URH_SC_HD __device__ __forceinline__
#define URH_DMUL(a, b) __dmul_rn((a), (b))
#define URH_DFMA(a, b, c) __fma_rn((a), (b), (c))
#define URH_D2I_RZ(x) __double2int_rz(x)
#define URH_D2F(x) __double2float_rn(x)
#define URH_SC_F2U(x) __float_as_uint(x)
#else
#if defined(__CUDACC__)
#define URH_SC_HD __host__ __device__ inline
#else
#define URH_SC_HD static inline
#endif
#define URH_DMUL(a, b) ((a) * (b))
#define URH_DFMA(a, b, c) fma((a), (b), (c))
#define URH_D2I_RZ(x) ((int32_t)(x))
#define URH_D2F(x) ((float)(x))
static inline uint32_t urh_sc_f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
#define URH_SC_F2U(x) urh_sc_f2u(x)
#endif

#define URH_SC_HPI_INV 0x1.45f306dc9c883p+23
#define URH_SC_HPI 0x1.921fb54442d18p+0
#define URH_SC_C1 -0x1.ffffffd0c621cp-2
#define URH_SC_C2 0x1.55553e1068f19p-5
#define URH_SC_C3 -0x1.6c087e89a359dp-10
#define URH_SC_C4 0x1.99343027bf8c3p-16
#define URH_SC_S1 -0x1.555545995a603p-3
#define URH_SC_S2 0x1.1107605230bc4p-7
#define URH_SC_S3 -0x1.994eb3774cf24p-13

// sine polynomial on (x*sign, x^2): s = fma(x3, S1, x); result = fma(fma(S3, x2, S2), x3*x2, s)
URH_SC_HD float urh_sc_sin_poly(double xs, double x2) {
    const double s1p = URH_DFMA(URH_SC_S3, x2, URH_SC_S2);
    const double x3 = URH_DMUL(x2, xs);
    const double x5 = URH_DMUL(x2, x3);
    const double s = URH_DFMA(x3, URH_SC_S1, xs);
    return URH_D2F(URH_DFMA(s1p, x5, s));
}
// cosine polynomial; neg = use table[1] (all cosine coefficients negated)
URH_SC_HD float urh_sc_cos_poly(double x2, int neg) {
    const double sg = neg ? -1.0 : 1.0;
    const double x4 = URH_DMUL(x2, x2);
    const double c1p = URH_DFMA(sg * URH_SC_C1, x2, sg);
    const double c2p = URH_DFMA(sg * URH_SC_C4, x2, sg * URH_SC_C3);
    const double x6 = URH_DMUL(x2, x4);
    const double c = URH_DFMA(x4, sg * URH_SC_C2, c1p);
    return URH_D2F(URH_DFMA(c2p, x6, c));
}

// 4/pi in 32-bit words, __inv_pio4[24] of s_sincosf_data.c — read from libm.so.6 .rodata at 0xb80c0
#if defined(__CUDA_ARCH__)
#define URH_SC_TABLE static __device__ const
#else
#define URH_SC_TABLE static const
#endif
URH_SC_TABLE uint32_t urh_inv_pio4[24] = {
    0x000000a2, 0x0000a2f9, 0x00a2f983, 0xa2f9836e, 0xf9836e4e, 0x836e4e44, 0x6e4e4415, 0x4e441529,
    0x441529fc, 0x1529fc27, 0x29fc2757, 0xfc2757d1, 0x2757d1f5, 0x57d1f534, 0xd1f534dd, 0xf534ddc0,
    0x34ddc0db, 0xddc0db62, 0xc0db6295, 0xdb629599, 0x6295993c, 0x95993c43, 0x993c4390, 0x3c439041};
#define URH_SC_PI63 0x1.921fb54442d18p-62

// reduce_large (code at 0x7e92b of the FMA sinf): x mod pi/2 for 120 <= |x| < inf, quadrant in *np
URH_SC_HD double urh_sc_reduce_large(uint32_t xi, int* np) {
    const uint32_t* arr = &urh_inv_pio4[(xi >> 26) & 15];
    const int shift = (xi >> 23) & 7;
    const uint32_t m = ((xi & 0x7fffffu) | 0x800000u) << shift;
    const uint32_t r0 = m * arr[0];
    const uint64_t res1 = (uint64_t)m * arr[4];
    const uint64_t res2 = (uint64_t)m * arr[8];
    uint64_t res0 = (res2 >> 32) | ((uint64_t)r0 << 32);
    res0 += res1;
    const uint64_t n = (res0 + (1ull << 61)) >> 62;
    res0 -= n << 62;
    *np = (int)n;
    return URH_DMUL((double)(int64_t)res0, URH_SC_PI63);
}

// *ok = 0 only for inf / nan
URH_SC_HD void urh_glibc_sincosf(float y, float* sn, float* cs, int* ok) {
    const uint32_t top = (URH_SC_F2U(y) >> 20) & 0x7ff;
    const double x = (double)y;
    *ok = 1;
    if (top <= 0x3f3) {  // |y| < pi/4
        if (top <= 0x397) {  // |y| < 2^-12
            *sn = y;
            *cs = 1.0f;
            return;
        }
        const double x2 = URH_DMUL(x, x);
        *sn = urh_sc_sin_poly(x, x2);
        *cs = urh_sc_cos_poly(x2, 0);
        return;
    }
    if (top > 0x42e) {  // |y| >= 120
        if (top >= 0x7f8) {  // inf / nan
            *ok = 0;
            *sn = 0.0f;
            *cs = 0.0f;
            return;
        }
        const uint32_t xi = URH_SC_F2U(y);
        int n;
        const double xr = urh_sc_reduce_large(xi, &n);
        const int ns = n + (int)(xi >> 31);
        const int neg = (ns & 2) ? 1 : 0;
        const double sign = ((ns & 3) == 1 || (ns & 3) == 2) ? -1.0 : 1.0;
        const double x2 = URH_DMUL(xr, xr);
        const double xs = URH_DMUL(xr, sign);
        if (n & 1) {
            *sn = urh_sc_cos_poly(x2, neg);
            *cs = urh_sc_sin_poly(xs, x2);
        } else {
            *sn = urh_sc_sin_poly(xs, x2);
            *cs = urh_sc_cos_poly(x2, neg);
        }
        return;
    }
    const double r = URH_DMUL(x, URH_SC_HPI_INV);
    const int32_t n = (URH_D2I_RZ(r) + 0x800000) >> 24;
    const double xr = URH_DFMA(-(double)n, URH_SC_HPI, x);  // vfnmadd: x - n*hpi, one rounding
    const double x2 = URH_DMUL(xr, xr);
    const int neg = (n & 2) ? 1 : 0;
    const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
    const double xs = URH_DMUL(xr, sign);
    // sinf uses polynomial n, cosf uses polynomial n^1 (odd -> cosine polynomial)
    if (n & 1) {
        *sn = urh_sc_cos_poly(x2, neg);
        *cs = urh_sc_sin_poly(xs, x2);
    } else {
        *sn = urh_sc_sin_poly(xs, x2);
        *cs = urh_sc_cos_poly(x2, neg);
    }
}
