// The dense (sample-rate) pass shared by demodulation, digitizing and message segmentation.
//
// Layout: the sample stream is cut into TILES of URH_TILE consecutive samples, one warp per tile.
// A warp walks its tile 64 samples at a time; lane l owns samples (2l, 2l+1) of each 64-group, i.e.
// one 128-bit load of two float2 IQ samples (fully coalesced: 512 B per warp per step) and one 64-bit
// store of two demodulated floats.  The FSK predecessor sample comes from the neighbouring lane by
// shuffle, never from a second load.
//
// The digitizer state machine of the reference (signal_functions.pyx:431-483) is restated in terms of
// RUNS of equal class (DESIGN.md §digitizer): a run produces a CANDIDATE at run_start + tolerance iff
// it is longer than `tolerance`.  Class boundaries are found with warp ballots, and the (warp-uniform)
// boundary bit-mask is walked by the whole warp in lock-step, so the per-sample cost of the state
// machine is two compares and two votes.  Runs that touch a tile edge are summarised (class, length)
// and stitched by a scan over the tile table (digitize.cu), which makes the decomposition exact for
// any tolerance.
#pragma once
#include "common.cuh"
#include "fdlibm_atan2f.h"

#define URH_TILE 2048          // samples per warp-tile (multiple of 64, < 65536)
#define URH_WARPS_PER_BLOCK 8
#define URH_MAX_THR 255

struct UrhClassify {
    float noise_value;     // exact-equality sentinel (signal_functions.pyx:435)
    int order;             // 2**bits_per_symbol
    float thr[URH_MAX_THR];  // get_center_thresholds (signal_functions.pyx:380-390)
};

struct __align__(16) UrhTileSummary {
    int16_t first_cls;
    int16_t last_cls;
    int32_t head_len;   // length of the run containing the tile's first sample (== tile_len if whole)
    int32_t tail_len;   // length (inside the tile) of the run containing the tile's last sample
    int32_t ncand;      // interior candidates written to the staging area
};

// Per-tile statistics of the demodulated samples that detect_center keeps (rect > -4, AutoInterpretation.py:227):
// produced by the dense pass so that the center histogram is the only extra pass over qad.
struct __align__(16) UrhTileStats {
    double sum, sumsq;
    float mn, mx;
    int32_t cnt;
    int32_t all_noise;   // 1: every sample of the tile equals the NOISE sentinel (the digitizer's class -1 throughout)
};

struct UrhStatAcc {
    double sum, sumsq;
    float mn, mx;
    int cnt;
    bool all_noise;
    __device__ __forceinline__ void init() { sum = 0.0; sumsq = 0.0; mn = INFINITY; mx = -INFINITY; cnt = 0; all_noise = true; }
    __device__ __forceinline__ void add(float v) {
        if (v > -4.0f) {
            const double d = (double)v;
            sum += d;
            sumsq += d * d;
            mn = fminf(mn, v);
            mx = fmaxf(mx, v);
            cnt++;
        }
    }
    // warp reduction, lane 0 writes
    __device__ __forceinline__ void store(UrhTileStats* out, int lane) {
        for (int off = 16; off > 0; off >>= 1) {
            sum += __shfl_down_sync(URH_FULL_MASK, sum, off);
            sumsq += __shfl_down_sync(URH_FULL_MASK, sumsq, off);
            mn = fminf(mn, __shfl_down_sync(URH_FULL_MASK, mn, off));
            mx = fmaxf(mx, __shfl_down_sync(URH_FULL_MASK, mx, off));
            cnt += __shfl_down_sync(URH_FULL_MASK, cnt, off);
        }
        const int alln = __all_sync(URH_FULL_MASK, all_noise) ? 1 : 0;
        if (lane == 0) {
            UrhTileStats t;
            t.sum = sum; t.sumsq = sumsq; t.mn = mn; t.mx = mx; t.cnt = cnt; t.all_noise = alln;
            *out = t;
        }
    }
};

// ---- IQ sample access ------------------------------------------------------------------------------
// (a + ib)(c + id) as std::complex<float> multiplies without -ffast-math (GCC): the naive product, and when both of its
// parts are NaN, libgcc's __mulsc3 recovery of C99 Annex G (an infinite operand gives an infinite result, not NaN).  The
// Costas loop (signal_functions.pyx:302) reaches the recovery on samples with an infinite imaginary part.
__device__ __forceinline__ void urh_cmulf(float a, float b, float c, float d, float& re, float& im) {
    const float ac = __fmul_rn(a, c), bd = __fmul_rn(b, d), ad = __fmul_rn(a, d), bc = __fmul_rn(b, c);
    re = __fsub_rn(ac, bd);
    im = __fadd_rn(ad, bc);
    if (isnan(re) && isnan(im)) {
        bool recalc = false;
        if (isinf(a) || isinf(b)) {
            a = copysignf(isinf(a) ? 1.0f : 0.0f, a);
            b = copysignf(isinf(b) ? 1.0f : 0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = true;
        }
        if (isinf(c) || isinf(d)) {
            c = copysignf(isinf(c) ? 1.0f : 0.0f, c);
            d = copysignf(isinf(d) ? 1.0f : 0.0f, d);
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            recalc = true;
        }
        if (!recalc && (isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc))) {
            if (isnan(a)) a = copysignf(0.0f, a);
            if (isnan(b)) b = copysignf(0.0f, b);
            if (isnan(c)) c = copysignf(0.0f, c);
            if (isnan(d)) d = copysignf(0.0f, d);
            recalc = true;
        }
        if (recalc) {
            re = __fmul_rn(INFINITY, __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, d)));
            im = __fmul_rn(INFINITY, __fadd_rn(__fmul_rn(a, d), __fmul_rn(b, c)));
        }
    }
}

template <int DT> struct UrhElem;
template <> struct UrhElem<URH_DT_I8> { typedef int8_t type; };
template <> struct UrhElem<URH_DT_U8> { typedef uint8_t type; };
template <> struct UrhElem<URH_DT_I16> { typedef int16_t type; };
template <> struct UrhElem<URH_DT_U16> { typedef uint16_t type; };
template <> struct UrhElem<URH_DT_F32> { typedef float type; };

struct UrhPair {
    float r0, i0, r1, i1;
};

__device__ __forceinline__ float4 urh_ldg_f4(const void* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ uint2 urh_ldg_u2(const void* p) {
    uint2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t urh_ldg_u1(const void* p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void urh_stg_f2(float* p, float a, float b) {
    asm volatile("st.global.L1::no_allocate.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// Load samples (i, i+1) of an (n,2) array.  `vec` = base pointer is aligned for a two-sample vector load.
template <int DT>
__device__ __forceinline__ UrhPair urh_load_pair(const void* base, int64_t i, int64_t n, bool vec) {
    typedef typename UrhElem<DT>::type E;
    const E* p = (const E*)base + 2 * i;
    UrhPair o;
    o.r0 = o.i0 = o.r1 = o.i1 = 0.0f;
    if (i + 1 < n && vec) {
        if (DT == URH_DT_F32) {
            const float4 v = urh_ldg_f4(p);
            o.r0 = v.x; o.i0 = v.y; o.r1 = v.z; o.i1 = v.w;
        } else if (DT == URH_DT_I16) {
            const uint2 v = urh_ldg_u2(p);
            o.r0 = (float)(int16_t)(v.x & 0xffff); o.i0 = (float)(int16_t)(v.x >> 16);
            o.r1 = (float)(int16_t)(v.y & 0xffff); o.i1 = (float)(int16_t)(v.y >> 16);
        } else if (DT == URH_DT_U16) {
            const uint2 v = urh_ldg_u2(p);
            o.r0 = (float)(v.x & 0xffff); o.i0 = (float)(v.x >> 16);
            o.r1 = (float)(v.y & 0xffff); o.i1 = (float)(v.y >> 16);
        } else if (DT == URH_DT_I8) {
            const uint32_t v = urh_ldg_u1(p);
            o.r0 = (float)(int8_t)(v & 0xff); o.i0 = (float)(int8_t)((v >> 8) & 0xff);
            o.r1 = (float)(int8_t)((v >> 16) & 0xff); o.i1 = (float)(int8_t)(v >> 24);
        } else {
            const uint32_t v = urh_ldg_u1(p);
            o.r0 = (float)(v & 0xff); o.i0 = (float)((v >> 8) & 0xff);
            o.r1 = (float)((v >> 16) & 0xff); o.i1 = (float)(v >> 24);
        }
    } else {
        if (i < n) { o.r0 = (float)__ldg(p); o.i0 = (float)__ldg(p + 1); }
        if (i + 1 < n) { o.r1 = (float)__ldg(p + 2); o.i1 = (float)__ldg(p + 3); }
    }
    return o;
}

// ---- demodulation of one sample (bit-faithful to signal_functions.pyx:363-376) ---------------------
struct UrhDemodParams {
    float noise_sqrd;   // noise_mag * noise_mag (float)
    float noise_value;  // NOISE sentinel
    float max_mag;      // ASK normalisation (pyx:343-352)
    float one, mone;    // +1.0f / -1.0f as run-time values (see fsk_fast.cuh: keeps ptxas from contracting)
};

// Per-sample terms of the reference's std::complex<float> expression
//   tmp = (x[i-1].re - 1j*x[i-1].im) * (x[i].re + 1j*x[i].im)
// with 1j*v = (0*v - 1*0, 0*0 + 1*v) and real -/+ complex acting on (real, 0); signed zeros matter.
// For a sample (re, im):   zt = 0*im - 0
//   as the CURRENT factor :  C = re + zt,  D = 0 + im
//   as the PREVIOUS factor:  A = re - zt,  B = 0 - (0 + im) = 0 - D
// so each sample's four terms are computed once and (A, B) travel to the next sample.
struct UrhFskTerms {
    float A, B, C, D;
};
__device__ __forceinline__ UrhFskTerms urh_fsk_terms(float re, float im) {
    UrhFskTerms t;
    const float zt = __fsub_rn(__fmul_rn(0.0f, im), 0.0f);
    t.C = __fadd_rn(re, zt);
    t.A = __fsub_rn(re, zt);
    t.D = __fadd_rn(0.0f, im);
    t.B = __fsub_rn(0.0f, t.D);
    return t;
}
// atan2f(imag, real) of (A + iB)(C + iD), bit-faithful to signal_functions.pyx:375-376
__device__ __forceinline__ float urh_fsk_angle(float A, float B, float C, float D) {
    const float xr = __fsub_rn(__fmul_rn(A, C), __fmul_rn(B, D));
    const float xi = __fadd_rn(__fmul_rn(A, D), __fmul_rn(B, C));
    return urh_atan2f_v2(xi, xr);
}

// ---- classification (signal_functions.pyx:435-442) --------------------------------------------------
__device__ __forceinline__ int urh_classify(float s, const UrhClassify& C) {
    if (s == C.noise_value) return -1;
    if (C.order == 2) return (s <= C.thr[0]) ? 0 : 1;
    int c = C.order - 1;
    for (int k = 0; k < C.order - 1; k++) {
        if (s <= C.thr[k]) { c = k; break; }
    }
    return c;
}

// ---- warp-uniform run tracker -------------------------------------------------------------------------
__device__ __forceinline__ uint64_t urh_spread_bits(uint32_t x) {
    uint64_t v = x;
    v = (v | (v << 16)) & 0x0000FFFF0000FFFFull;
    v = (v | (v << 8)) & 0x00FF00FF00FF00FFull;
    v = (v | (v << 4)) & 0x0F0F0F0F0F0F0F0Full;
    v = (v | (v << 2)) & 0x3333333333333333ull;
    v = (v | (v << 1)) & 0x5555555555555555ull;
    return v;
}

struct UrhRunTracker {
    int tol;
    int run_start, run_cls, first_cls, head_len, ncand, carry_cls;
    bool is_head;
    uint32_t cm_n, cm_a;   // feed_masks: the open run's class bits as full words
    uint32_t* stage;   // this tile's staging slots

    __device__ __forceinline__ void init(int tol_, uint32_t* stage_) {
        tol = tol_; stage = stage_;
        run_start = 0; run_cls = -2; first_cls = -2; head_len = 0; ncand = 0; carry_cls = -2; is_head = true;
        cm_n = 0xffffffffu; cm_a = 0xffffffffu;
    }
    __device__ __forceinline__ void emit(int pos, int cls, int lane) {
        if (lane == 0) stage[ncand] = ((uint32_t)pos << 16) | (uint32_t)(cls + 1);
        ncand++;
    }
    // c0,c1: classes of this lane's two samples of 64-group `it`; v0,v1: sample exists (inside the tile)
    __device__ __forceinline__ void feed(int it, int c0, int c1, bool v0, bool v1, int lane) {
        int pc = __shfl_up_sync(URH_FULL_MASK, c1, 1);
        if (lane == 0) pc = carry_cls;
        const bool b0 = v0 && (c0 != pc);
        const bool b1 = v1 && (c1 != c0);
        carry_cls = __shfl_sync(URH_FULL_MASK, c1, 31);
        const uint32_t m0 = __ballot_sync(URH_FULL_MASK, b0);
        const uint32_t m1 = __ballot_sync(URH_FULL_MASK, b1);
        if ((m0 | m1) == 0u) return;
        walk(it, m0, m1, c0, c1, lane);
    }
    // Binary classifiers (one threshold): the classes of a 64-group as four WARP MASKS - n0/n1: sample 2l / 2l+1 is noise (class -1),
    // a0/a1: it is above the threshold (never set together with the noise bit).  The boundary masks are bit arithmetic on the masks:
    // warp-uniform work (no shuffles, no per-lane class integers), the per-lane classes are only formed when a boundary exists.
    // Full 64-groups only; do not mix with feed() inside one tile (feed() carries the previous class in carry_cls, this one in run_cls).
    __device__ __forceinline__ void feed_masks(int it, uint32_t n0, uint32_t a0, uint32_t n1, uint32_t a1, int lane) {
        // no boundary <=> all 64 samples repeat the open run's class: cm_n / cm_a are that class's bits spread over a word (the
        // impossible pair ~0 / ~0 before the tile's first sample, so the first group always takes the long way)
        if ((((n0 ^ cm_n) | (n1 ^ cm_n)) | ((a0 ^ cm_a) | (a1 ^ cm_a))) == 0u) return;
        // class bits of the sample before sample 2l: sample 2(l-1)+1, for lane 0 the previous group's last sample
        uint32_t m0 = (((n1 << 1) | (cm_n & 1u)) ^ n0) | (((a1 << 1) | (cm_a & 1u)) ^ a0);
        if (run_cls == -2) m0 |= 1u;                    // the tile's first sample opens the head run
        uint32_t m1 = (n0 ^ n1) | (a0 ^ a1);
        feed_masks_slow(it, n0, a0, n1, a1, m0, m1, lane);
        cm_n = (run_cls < 0) ? 0xffffffffu : 0u;
        cm_a = (run_cls == 1) ? 0xffffffffu : 0u;
    }
    __device__ __forceinline__ void feed_masks_slow(int it, uint32_t n0, uint32_t a0, uint32_t n1, uint32_t a1, uint32_t m0, uint32_t m1,
                                                    int lane) {
        const int nb = __popc(m0) + __popc(m1);
        if (nb == 1 && run_cls != -2 && !is_head) {
            // the common case of a demodulated signal (one symbol edge in 64 samples, inside the tile): no loop
            const bool take0 = m0 != 0u;
            const int l = __ffs(m0 | m1) - 1;
            const int p = it * 64 + 2 * l + (take0 ? 0 : 1);
            const uint32_t nbit = ((take0 ? n0 : n1) >> l) & 1u, abit = ((take0 ? a0 : a1) >> l) & 1u;
            if (p - run_start > tol) emit(run_start + tol, run_cls, lane);
            run_start = p;
            run_cls = nbit ? -1 : (int)abit;
            return;
        }
        if (nb > 4) {
            const int c0 = ((n0 >> lane) & 1u) ? -1 : (int)((a0 >> lane) & 1u);
            const int c1 = ((n1 >> lane) & 1u) ? -1 : (int)((a1 >> lane) & 1u);
            walk_parallel(it, m0, m1, c0, c1, lane);
            return;
        }
        while (m0 | m1) {
            const int l0 = m0 ? (__ffs(m0) - 1) : 64;
            const int l1 = m1 ? (__ffs(m1) - 1) : 64;
            const bool take0 = l0 <= l1;
            const int l = take0 ? l0 : l1;
            if (take0) m0 &= m0 - 1; else m1 &= m1 - 1;
            const int p = it * 64 + 2 * l + (take0 ? 0 : 1);
            const uint32_t nbit = ((take0 ? n0 : n1) >> l) & 1u, abit = ((take0 ? a0 : a1) >> l) & 1u;
            const int cls_p = nbit ? -1 : (int)abit;
            if (run_cls == -2) {
                first_cls = cls_p;
            } else if (is_head) {
                head_len = p;
                is_head = false;
            } else if (p - run_start > tol) {
                emit(run_start + tol, run_cls, lane);
            }
            run_start = p;
            run_cls = cls_p;
        }
    }
    // Same as feed() but with the boundary predicates supplied by the caller (fsk_fast.cuh derives them
    // without materialising class integers for the compare).
    __device__ __forceinline__ void walk(int it, uint32_t m0, uint32_t m1, int c0, int c1, int lane) {
        // Few boundaries (a demodulated signal: one per symbol): walk them one by one, warp-uniformly.  Many boundaries (noise
        // that is not gated: a class change at almost every sample): every lane settles its own two samples at once.
        if (__popc(m0) + __popc(m1) > 4) {
            walk_parallel(it, m0, m1, c0, c1, lane);
            return;
        }
        // merge the two boundary masks in sample order: sample 2l (mask m0) precedes sample 2l+1 (mask m1)
        while (m0 | m1) {
            const int l0 = m0 ? (__ffs(m0) - 1) : 64;
            const int l1 = m1 ? (__ffs(m1) - 1) : 64;
            const bool take0 = l0 <= l1;
            const int l = take0 ? l0 : l1;
            if (take0) m0 &= m0 - 1; else m1 &= m1 - 1;
            const int p = it * 64 + 2 * l + (take0 ? 0 : 1);
            const int cls_p = __shfl_sync(URH_FULL_MASK, take0 ? c0 : c1, l);
            if (run_cls == -2) {
                first_cls = cls_p;                    // the forced boundary at p == 0 opens the head run
            } else if (is_head) {
                head_len = p;
                is_head = false;
            } else if (p - run_start > tol) {
                emit(run_start + tol, run_cls, lane);
            }
            run_start = p;
            run_cls = cls_p;
        }
    }
    // The same bookkeeping with O(1) work per 64-group, however many boundaries it holds.  A boundary at position p closes the
    // run [q, p) that its PREDECESSOR boundary q opened (q = the nearest boundary below p in this group, else the carried
    // run_start); the run's class is the class of sample p - 1.  The run emits a candidate at q + tol iff it is longer than tol
    // and is not the tile's head run (the run that starts at the tile's first sample, handled by the tile stitching).
    __device__ __forceinline__ void walk_parallel(int it, uint32_t m0, uint32_t m1, int c0, int c1, int lane) {
        const uint32_t lt = (1u << lane) - 1u;
        const int base = it * 64;
        // class of the sample before each of my two samples
        int cprev0 = __shfl_up_sync(URH_FULL_MASK, c1, 1);
        if (lane == 0) cprev0 = run_cls;   // the carried run's class (== class of the previous group's last sample)
        const int cprev1 = c0;
        // nearest boundary below sample (l, 0): among m1 at lanes < l (position 2l'+1) and m0 at lanes < l (position 2l')
        const uint32_t b1 = m1 & lt, b0 = m0 & lt;
        int q0 = -1;   // relative to `base`; -1 = none in this group
        if (b1) q0 = 2 * (31 - __clz(b1)) + 1;
        if (b0) q0 = max(q0, 2 * (31 - __clz(b0)));
        const bool has0 = (m0 >> lane) & 1u, has1 = (m1 >> lane) & 1u;
        const int q1 = has0 ? 2 * lane : q0;
        // absolute start of the run each of my boundaries closes, and whether that run is the head run
        const bool carried_head = is_head;                 // the carried run (if any) is the head run
        const int start0 = (q0 >= 0) ? base + q0 : run_start;
        const int start1 = (q1 >= 0) ? base + q1 : run_start;
        const int p0 = base + 2 * lane, p1 = p0 + 1;
        // a run opened inside this group is the head run only if it starts at the tile's first sample (p == 0, it == 0)
        const bool head0 = (q0 >= 0) ? (start0 == 0) : (carried_head || run_cls == -2);
        const bool head1 = (q1 >= 0) ? (start1 == 0) : (carried_head || run_cls == -2);
        const bool emit0 = has0 && !head0 && (p0 - start0 > tol);
        const bool emit1 = has1 && !head1 && (p1 - start1 > tol);
        const uint32_t e0 = __ballot_sync(URH_FULL_MASK, emit0), e1 = __ballot_sync(URH_FULL_MASK, emit1);
        const int before = __popc(e0 & lt) + __popc(e1 & lt);
        if (emit0) stage[ncand + before] = ((uint32_t)(start0 + tol) << 16) | (uint32_t)(cprev0 + 1);
        if (emit1) stage[ncand + before + (emit0 ? 1 : 0)] = ((uint32_t)(start1 + tol) << 16) | (uint32_t)(cprev1 + 1);
        ncand += __popc(e0) + __popc(e1);
        // head run: it ends at the first boundary of the tile that is not the tile-opening one at p == 0
        uint32_t f0 = m0, f1 = m1;
        if (run_cls == -2) {   // the tile's first group: the forced boundary at p == 0 opens the head run
            first_cls = __shfl_sync(URH_FULL_MASK, c0, 0);
            f0 &= ~1u;
        }
        if (is_head && (f0 | f1)) {
            const int l0 = f0 ? (__ffs(f0) - 1) : 64, l1 = f1 ? (__ffs(f1) - 1) : 64;
            head_len = base + ((l0 <= l1) ? 2 * l0 : 2 * l1 + 1);
            is_head = false;
        }
        // carry: the last boundary of the group opens the run that continues into the next group
        const int h0 = m0 ? (31 - __clz(m0)) : -1, h1 = m1 ? (31 - __clz(m1)) : -1;
        const bool last_is_1 = h1 >= h0;   // position 2*h1+1 > 2*h0 whenever h1 >= h0
        const int hl = last_is_1 ? h1 : h0;
        run_start = base + 2 * hl + (last_is_1 ? 1 : 0);
        run_cls = __shfl_sync(URH_FULL_MASK, last_is_1 ? c1 : c0, hl);
    }
    __device__ __forceinline__ void finish(int tile_len, UrhTileSummary* out, int lane) {
        if (is_head) head_len = tile_len;
        else if (tile_len - run_start > tol) emit(run_start + tol, run_cls, lane);
        if (lane == 0) {
            UrhTileSummary s;
            s.first_cls = (int16_t)first_cls;
            s.last_cls = (int16_t)run_cls;
            s.head_len = head_len;
            s.tail_len = tile_len - run_start;
            s.ncand = ncand;
            *out = s;
        }
    }
};

// ---- whole-tile resolve for binary classifiers ---------------------------------------------------------------------------------
// A FULL tile is 32 groups of 64 samples, and a warp has 32 lanes: while the tile streams through, lane g keeps group g's class
// masks (UrhRunTracker::feed_masks' n0/a0/n1/a1); afterwards every lane settles the boundaries of ITS group, with one prefix-max
// over the lanes for "where did the run that enters my group start" and one prefix-sum for the candidates' slots.  The work per
// tile no longer depends on how the boundaries are spread (one loop iteration per boundary of the busiest group), the streaming
// loop holds no bookkeeping at all, and the code is a fraction of the inlined group-by-group walk (instruction cache).
// Same results as UrhRunTracker: a boundary at p closes the run [q, p) opened by its predecessor q; the run that starts at the
// tile's first sample is the head run (head_len, no candidate); any other run longer than tol leaves the candidate (q + tol, class).
struct UrhTileResolve {
    uint32_t n0, a0, n1, a1;   // this lane's group
    __device__ __forceinline__ void init() { n0 = a0 = n1 = a1 = 0u; }
    __device__ __forceinline__ void keep(int g, uint32_t gn0, uint32_t ga0, uint32_t gn1, uint32_t ga1, int lane) {
        if (lane == g) { n0 = gn0; a0 = ga0; n1 = gn1; a1 = ga1; }
    }
    __device__ __forceinline__ static int cls_of(uint32_t nbit, uint32_t abit) { return (nbit & 1u) ? -1 : (int)(abit & 1u); }

    template <bool WRITE>
    __device__ __forceinline__ int walk(uint32_t m0, uint32_t m1, uint32_t pn, uint32_t pa, int q, int tol, int lane, uint32_t* dst) const {
        int k = 0;
        const int base = lane * 64;
        while (m0 | m1) {
            const int l0 = m0 ? (__ffs(m0) - 1) : 64;
            const int l1 = m1 ? (__ffs(m1) - 1) : 64;
            const bool take0 = l0 <= l1;
            const int l = take0 ? l0 : l1;
            if (take0) m0 &= m0 - 1; else m1 &= m1 - 1;
            const int p = base + 2 * l + (take0 ? 0 : 1);
            if (q > 0 && p - q > tol) {      // q == 0: the head run; q < 0: p is the tile's first sample
                if (WRITE) {
                    // the closed run's class = the class of sample p - 1
                    uint32_t nb, ab;
                    if (!take0) { nb = n0 >> l; ab = a0 >> l; }
                    else if (l > 0) { nb = n1 >> (l - 1); ab = a1 >> (l - 1); }
                    else { nb = pn; ab = pa; }
                    dst[k] = ((uint32_t)(q + tol) << 16) | (uint32_t)(cls_of(nb, ab) + 1);
                }
                k++;
            }
            q = p;
        }
        return k;
    }

    // tile_len == URH_TILE.  stage: this tile's staging slots.
    __device__ __forceinline__ void finish(int tol, uint32_t* stage, UrhTileSummary* out, int lane) const {
        // class bits of the sample before my group's first sample
        const uint32_t pn = __shfl_up_sync(URH_FULL_MASK, n1 >> 31, 1), pa = __shfl_up_sync(URH_FULL_MASK, a1 >> 31, 1);
        uint32_t m0 = (((n1 << 1) | (pn & 1u)) ^ n0) | (((a1 << 1) | (pa & 1u)) ^ a0);
        if (lane == 0) m0 |= 1u;   // the tile's first sample opens the head run
        const uint32_t m1 = (n0 ^ n1) | (a0 ^ a1);
        int last = -1;             // my group's last boundary (tile-relative)
        if (m1) last = lane * 64 + 2 * (31 - __clz(m1)) + 1;
        if (m0) last = max(last, lane * 64 + 2 * (31 - __clz(m0)));
        int incl = last;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int t = __shfl_up_sync(URH_FULL_MASK, incl, off);
            if (lane >= off) incl = max(incl, t);
        }
        int q = __shfl_up_sync(URH_FULL_MASK, incl, 1);   // where the run entering my group started
        if (lane == 0) q = -1;
        const int L = __shfl_sync(URH_FULL_MASK, incl, 31);   // the tile's last boundary (>= 0: the one at sample 0)
        // head run: ends at the first boundary after sample 0
        uint32_t f0 = m0, f1 = m1;
        if (lane == 0) f0 &= ~1u;
        int first = URH_TILE;
        if (f0 | f1) {
            const int l0 = f0 ? (__ffs(f0) - 1) : 64, l1 = f1 ? (__ffs(f1) - 1) : 64;
            first = lane * 64 + ((l0 <= l1) ? 2 * l0 : 2 * l1 + 1);
        }
        const int head_len = __reduce_min_sync(URH_FULL_MASK, first);
        // candidates: count, slot, write
        const int mine = walk<false>(m0, m1, pn, pa, q, tol, lane, nullptr);
        int pre = mine;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int t = __shfl_up_sync(URH_FULL_MASK, pre, off);
            if (lane >= off) pre += t;
        }
        int total = __shfl_sync(URH_FULL_MASK, pre, 31);
        if (mine) walk<true>(m0, m1, pn, pa, q, tol, lane, stage + (pre - mine));
        // the run that is still open at the tile's end
        const int last_cls = __shfl_sync(URH_FULL_MASK, cls_of(n1 >> 31, a1 >> 31), 31);
        if (L > 0 && URH_TILE - L > tol) {
            if (lane == 0) stage[total] = ((uint32_t)(L + tol) << 16) | (uint32_t)(last_cls + 1);
            total++;
        }
        if (lane == 0) {
            UrhTileSummary s;
            s.first_cls = (int16_t)cls_of(n0, a0);
            s.last_cls = (int16_t)last_cls;
            s.head_len = head_len;
            s.tail_len = URH_TILE - L;
            s.ncand = total;
            *out = s;
        }
    }
};
