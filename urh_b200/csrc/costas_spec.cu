// Speculative, chunk-parallel Costas loop — bit-identical to the serial recurrence of the reference
// (signal_functions.pyx:252-330), SURVEY hard part H2.
//
// The PLL is contracting: two trajectories that sit in the same lock branch (phase offsets of 2*pi/order apart)
// become BITWISE identical after a few hundred non-noise samples (measured on the CPU with glibc arithmetic:
// >99 % of the starts inside a burst merge within 300 samples).  Hence:
//   pass 1  (parallel: one thread per chunk and per branch candidate): start W samples before the chunk from the
//           loop's initial state rotated by k*2*pi/order, run through the chunk, write the outputs to candidate
//           buffer k and the loop state at every 256-sample checkpoint;
//   pass 2  (one warp, chained): carry the TRUE state from chunk to chunk.  If it equals a candidate's state at the
//           chunk start (bitwise), that candidate's run IS the true run for the whole chunk: O(1).  Otherwise step
//           the true state serially through the chunk, segment by segment, until it meets a candidate checkpoint
//           bitwise (typically ~300 samples after a burst starts); all-noise segments are skipped in O(1) because the
//           loop state is frozen on noise samples (pyx:293-295) and every candidate holds NOISE there;
//   pass 3  (parallel): assemble the result from the chosen candidate per segment.
// Nothing is accepted on similarity: a candidate's samples are used only downstream of a bitwise state match, where
// the deterministic recurrence guarantees identical results.  Worst case (never matching) degrades to the serial loop.
#include "dense.cuh"
#include "glibc_sincosf.h"

#include <math.h>
#include <stdlib.h>

#define CS_SEG 256
#define CS_MAX_SEGS 16          // chunk = segs * 256 samples, segs in {2,4,8,16} chosen from the capture length
#define CS_WARM 1024
#define CS_MAXBR 4
#define CS_STATS 6              // per stitch hypothesis: {O(1) chunks, walked chunks, samples stepped, self-chained, A, B}
// How a run starts (the `start` argument of the kernels below):
//   CS_EXACT  the true incoming loop state is known: chunk 0 has one exact run (from *st0, or the loop's initial {0, 1.5} when
//             st0 is NULL) and super-chunk 0 one chain;
//   CS_CAP    sample 0 is the capture's first sample: result[0] is not computed (written as 0) and warm-ups clip at index 1.
// A resident capture (and the first shard of a sharded one) has both, later shards neither, and the ring chunks c > 0 of a streamed
// capture only CS_EXACT: their incoming state is the preceding chunk's end state, left on the device.
#define CS_EXACT 1
#define CS_CAP 2

struct CsParams {
    float noise_sqrd, alpha, beta, scale, shift;
    int order;  // 2 or 4
    int segs;   // segments per chunk
    int chunk;  // samples per chunk = segs * CS_SEG
};

struct __align__(8) CsState {
    float freq, phase;
};

template <int DT>
__device__ __forceinline__ void cs_load(const void* iq, int64_t i, float& re, float& im) {
    typedef typename UrhElem<DT>::type E;
    const E* p = (const E*)iq + 2 * i;
    re = (float)p[0];
    im = (float)p[1];
}

// one sample of the loop; returns true if the sample is above the noise gate (state advanced), out = result[i]
__device__ __forceinline__ bool cs_step(CsState& s, float re, float im, const CsParams& P, float& out) {
    if (__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)) <= P.noise_sqrd) {
        out = -4.0f;
        return false;
    }
    const float rf = __fdiv_rn(__fadd_rn(re, P.shift), P.scale);
    const float jf = __fdiv_rn(__fadd_rn(im, P.shift), P.scale);
    const float cs_r = __fadd_rn(rf, __fmul_rn(0.0f, jf));          // rf + (0*jf - 1*0)
    const float cs_i = __fadd_rn(0.0f, __fadd_rn(0.0f, jf));
    float sn, cn;
    int ok;
    urh_glibc_sincosf(-s.phase, &sn, &cn, &ok);
    if (!ok) sincosf(-s.phase, &sn, &cn);
    const float nr = __fadd_rn(cn, __fmul_rn(0.0f, sn));
    const float ni = __fadd_rn(0.0f, __fadd_rn(0.0f, sn));
    float xr, xi;
    urh_cmulf(nr, ni, cs_r, cs_i, xr, xi);   // the products 1j*jf and 1j*sin never reach the Annex G recovery
    float err;
    if (P.order == 2) err = __fmul_rn(xi, xr);
    else {
        const float f1 = xr > 0.0f ? 1.0f : -1.0f;
        const float f2 = xi > 0.0f ? 1.0f : -1.0f;
        err = __fsub_rn(__fmul_rn(f1, xi), __fmul_rn(f2, xr));
    }
    err = err < -1.0f ? -1.0f : (err > 1.0f ? 1.0f : err);
    s.freq = __fadd_rn(s.freq, __fmul_rn(P.beta, err));
    s.phase = __fadd_rn(s.phase, __fadd_rn(s.freq, __fmul_rn(P.alpha, err)));
    const double two_pi = 2.0 * M_PI;
    while ((double)s.phase > two_pi) s.phase = (float)((double)s.phase - two_pi);
    while ((double)s.phase < -two_pi) s.phase = (float)((double)s.phase + two_pi);
    s.freq = s.freq < -1.0f ? -1.0f : (s.freq > 1.0f ? 1.0f : s.freq);
    out = (P.order == 2) ? xr : (float)(2.0 * (double)xr + (double)xi);
    return true;
}

// run the loop over samples [a, b): loads are issued four samples ahead of the dependent recurrence
template <int DT, bool WRITE>
__device__ __forceinline__ int cs_run(const void* iq, int64_t a, int64_t b, CsState& s, const CsParams& P, float* out, int) {
    int cnt = 0;
    float re[4], im[4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
        re[t] = im[t] = 0.f;
        if (a + t < b) cs_load<DT>(iq, a + t, re[t], im[t]);
    }
    for (int64_t i0 = a; i0 < b; i0 += 4) {
        float nre[4], nim[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
            nre[t] = nim[t] = 0.f;
            if (i0 + 4 + t < b) cs_load<DT>(iq, i0 + 4 + t, nre[t], nim[t]);
        }
#pragma unroll
        for (int t = 0; t < 4; t++) {
            if (i0 + t < b) {
                float o;
                cnt += cs_step(s, re[t], im[t], P, o) ? 1 : 0;
                if (WRITE) out[i0 + t] = o;
            }
        }
#pragma unroll
        for (int t = 0; t < 4; t++) { re[t] = nre[t]; im[t] = nim[t]; }
    }
    return cnt;
}

// pass 1: grid.x covers chunks, grid.y = candidate k
template <int DT>
__global__ void __launch_bounds__(128) k_cs_speculate(const void* __restrict__ iq, int64_t n, CsParams P, int64_t nchunks,
                                                      float* __restrict__ cand, CsState* __restrict__ ckpt,
                                                      int* __restrict__ nonnoise, int* __restrict__ chunk_cnt, int start,
                                                      const CsState* __restrict__ st0) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int k = blockIdx.y;
    if (c >= nchunks) return;
    const int64_t p0 = c * P.chunk;
    float* out = cand + (int64_t)k * n;
    CsState* ck = ckpt + ((int64_t)k * nchunks + c) * (P.segs + 1);
    CsState s;
    s.freq = 0.0f;
    // candidate k: the loop's initial phase 1.5 rotated by k * 2*pi/order (branch of the lock point)
    s.phase = (float)(1.5 + (double)k * (2.0 * M_PI / (double)P.order));
    if ((double)s.phase > 2.0 * M_PI) s.phase = (float)((double)s.phase - 2.0 * M_PI);
    float o;
    if (c == 0 && (start & CS_EXACT)) {
        if (k != 0) return;  // chunk 0 starts from the true incoming state: one exact run only
        if (st0) s = *st0;
        else s.phase = 1.5f;
    } else {
        // later shards of a sharded capture have CS_WARM halo samples stored in front of iq (negative indices); an exact start
        // has none and clips the warm-up at its first sample
        int64_t w0 = p0 - CS_WARM;
        const int64_t lo = (start & CS_CAP) ? 1 : 0;
        if ((start & CS_EXACT) && w0 < lo) w0 = lo;
        cs_run<DT, false>(iq, w0, p0, s, P, nullptr, 0);
    }
    ck[0] = s;
    int total = 0;
    for (int j = 0; j < P.segs; j++) {
        const int64_t a = p0 + (int64_t)j * CS_SEG;
        int64_t a0 = a;
        if (a0 == 0 && (start & CS_CAP)) { out[0] = 0.0f; a0 = 1; }  // the reference loop starts at i = 1 (result[0] undefined -> 0)
        const int64_t b0 = min(a + (int64_t)CS_SEG, n);
        const int cnt = cs_run<DT, true>(iq, a0, b0, s, P, out, 0);
        ck[j + 1] = s;
        total += cnt;
        if (k == 0) nonnoise[c * P.segs + j] = cnt;
    }
    if (k == 0) chunk_cnt[c] = total;
}

// ---- pass 2: the chain ------------------------------------------------------------------------------------------------
// A chain carries a loop state from chunk to chunk.  If the state equals a candidate's state at the chunk start (bitwise),
// that candidate's run IS the run for the whole chunk: O(1).  Otherwise the state is stepped through the chunk segment by
// segment until it meets a candidate checkpoint.  Tables (one set per chain family t):
//   src[t][c*segs + j]   candidate whose samples are right in that segment, or 255 = "stepped here"
//   segst[t][c*segs + j] the state at the start of a stepped segment (k_cs_fix recomputes those samples from it)
// The chain itself is still serial, so it is run speculatively as well (pass 2a): the chunks are grouped into super-chunks
// of T.sup chunks (>= 128 Ki samples) and one warp per (super-chunk, candidate k) runs the chain through the super-chunk ASSUMING it starts in
// candidate k's start state.  Pass 2b (one warp) then only hops from super-chunk to super-chunk: the true state at a
// super-chunk start almost always equals one of the assumptions (bitwise) -> take that chain's tables and end state; if
// not, the warp runs the chain through that super-chunk itself (table family nbr).  Exactness is by construction as in
// pass 1: a chain is only ever adopted when its starting state is bit-identical to the true one.
#define CS_SUP_MIN 64              // chunks per super-chunk, at least; raised so that a super-chunk spans >= 128 Ki samples

struct CsTables {
    uint8_t* src;     // [2 * nbr + 1][nseg]
    CsState* segst;   // [2 * nbr + 1][nseg]
    int64_t nseg;     // nchunks * segs
    int sup;          // chunks per super-chunk
};

// one warp; returns the state after chunk hi-1.  acc[0..2] += {O(1) chunks, walked chunks, samples stepped}
template <int DT>
__device__ CsState cs_chain(const void* __restrict__ iq, int64_t n, const CsParams& P, int64_t nchunks, int nbr,
                            const CsState* __restrict__ ckpt, const int* __restrict__ nonnoise, const int* __restrict__ chunk_cnt,
                            uint8_t* __restrict__ src, CsState* __restrict__ segst, int cap_start, int64_t lo, int64_t hi, CsState st,
                            int64_t* acc) {
    const int lane = threadIdx.x & 31;
    int64_t fast = 0, slow = 0, stepped = 0;
    for (int64_t c0 = lo; c0 < hi; c0 += 32) {
        // every lane prefetches the candidates' start/end states of chunk c0 + lane
        const int64_t cl = c0 + lane;
        CsState s0[CS_MAXBR], s1[CS_MAXBR];
#pragma unroll
        for (int k = 0; k < CS_MAXBR; k++) {
            if (k < nbr && cl < hi) {
                const CsState* ck = ckpt + ((int64_t)k * nchunks + cl) * (P.segs + 1);
                s0[k] = ck[0];
                s1[k] = ck[P.segs];
            } else {
                s0[k].freq = s0[k].phase = s1[k].freq = s1[k].phase = __int_as_float(0x7fc00000);
            }
        }
        const int my_cnt = (cl < hi) ? chunk_cnt[cl] : 0;
        const int todo = (int)min((int64_t)32, hi - c0);
        for (int t = 0; t < todo; t++) {
            const int64_t c = c0 + t;
            const int ccnt = __shfl_sync(URH_FULL_MASK, my_cnt, t);
            int match = -1;
            CsState e;
            e.freq = e.phase = 0.f;
#pragma unroll
            for (int k = 0; k < CS_MAXBR; k++) {
                const float f0 = __shfl_sync(URH_FULL_MASK, s0[k].freq, t), p0 = __shfl_sync(URH_FULL_MASK, s0[k].phase, t);
                const float f1 = __shfl_sync(URH_FULL_MASK, s1[k].freq, t), p1 = __shfl_sync(URH_FULL_MASK, s1[k].phase, t);
                if (match < 0 && k < nbr && __float_as_uint(f0) == __float_as_uint(st.freq) &&
                    __float_as_uint(p0) == __float_as_uint(st.phase)) {
                    match = k;
                    e.freq = f1;
                    e.phase = p1;
                }
            }
            if (match >= 0) {  // O(1): the candidate's run is the run
                if (lane < P.segs) src[c * P.segs + lane] = (uint8_t)match;
                st = e;
                fast++;
                continue;
            }
            if (ccnt == 0) {  // all-noise chunk: the loop state is frozen, every candidate holds NOISE
                if (lane < P.segs) src[c * P.segs + lane] = 0;
                fast++;
                continue;
            }
            slow++;
            // walk the chunk; lane 0 computes, the decision is broadcast
            int merged = -1, jm = P.segs;
            for (int j = 0; j < P.segs; j++) {
                const int cnt = nonnoise[c * P.segs + j];
                if (cnt == 0) {  // state frozen, every candidate holds NOISE here
                    if (lane == 0) src[c * P.segs + j] = 0;
                    continue;
                }
                if (lane == 0) {
                    src[c * P.segs + j] = 255;
                    segst[c * P.segs + j] = st;
                }
                const int64_t a = c * P.chunk + (int64_t)j * CS_SEG;
                // the warp stages the whole segment at once (8 coalesced loads in flight per lane) and evaluates the noise
                // gate in parallel; lane 0 then advances the loop over the non-noise samples only (the samples themselves
                // are written by k_cs_fix)
                float sre[CS_SEG / 32], sim[CS_SEG / 32];
                unsigned smask[CS_SEG / 32];
#pragma unroll
                for (int g = 0; g < CS_SEG / 32; g++) {
                    const int64_t i = a + g * 32 + lane;
                    sre[g] = 0.f; sim[g] = 0.f;
                    if (i < n && !(i == 0 && cap_start)) cs_load<DT>(iq, i, sre[g], sim[g]);
                }
#pragma unroll
                for (int g = 0; g < CS_SEG / 32; g++) {
                    const int64_t i = a + g * 32 + lane;
                    const bool live = (i < n && !(i == 0 && cap_start)) &&
                                      !(__fadd_rn(__fmul_rn(sre[g], sre[g]), __fmul_rn(sim[g], sim[g])) <= P.noise_sqrd);
                    smask[g] = __ballot_sync(URH_FULL_MASK, live);
                }
#pragma unroll
                for (int g = 0; g < CS_SEG / 32; g++) {
                    unsigned mask = smask[g];
                    while (mask) {
                        const int l = __ffs(mask) - 1;
                        mask &= mask - 1;
                        const float r1 = __shfl_sync(URH_FULL_MASK, sre[g], l), i1 = __shfl_sync(URH_FULL_MASK, sim[g], l);
                        if (lane == 0) {
                            float o;
                            cs_step(st, r1, i1, P, o);
                        }
                    }
                }
                stepped += cnt;
                st.freq = __shfl_sync(URH_FULL_MASK, st.freq, 0);
                st.phase = __shfl_sync(URH_FULL_MASK, st.phase, 0);
                // does the state now coincide with a candidate checkpoint?
                int m = -1;
                if (lane < nbr) {
                    const CsState q = ckpt[((int64_t)lane * nchunks + c) * (P.segs + 1) + j + 1];
                    if (__float_as_uint(q.freq) == __float_as_uint(st.freq) && __float_as_uint(q.phase) == __float_as_uint(st.phase)) m = lane;
                }
                const unsigned any = __ballot_sync(URH_FULL_MASK, m >= 0);
                if (any) {
                    merged = __ffs(any) - 1;
                    jm = j + 1;
                    break;
                }
            }
            if (merged >= 0) {
                if (lane >= jm && lane < P.segs) src[c * P.segs + lane] = (uint8_t)merged;
                const CsState q = ckpt[((int64_t)merged * nchunks + c) * (P.segs + 1) + P.segs];
                st = q;
            }
        }
    }
    acc[0] += fast; acc[1] += slow; acc[2] += stepped;
    return st;
}

// pass 2a: one warp per (super-chunk w, assumption k).  sup_end[w*nbr + k] = state after the super-chunk, sup_acc its counters.
// family 0 ("A"): the super-chunk starts in candidate k's start state (right whenever the loop is locked at its first sample).
// family 1 ("B"): it starts in the state family-A chain k of the last super-chunk WITH SIGNAL before it ended in -- right
//                 when the super-chunk starts inside a gap: the loop state is frozen there (or creeps on noise spikes), no
//                 candidate warm-up can reproduce it, but it is what the previous burst left behind.
template <int DT>
__global__ void __launch_bounds__(128) k_cs_chains(const void* __restrict__ iq, int64_t n, CsParams P, int64_t nchunks, int nbr,
                                                  const CsState* __restrict__ ckpt, const int* __restrict__ nonnoise,
                                                  const int* __restrict__ chunk_cnt, CsTables T, int start, int64_t nsuper,
                                                  int family, const int64_t* __restrict__ prev_live, const CsState* __restrict__ end_a,
                                                  CsState* __restrict__ sup_end, int64_t* __restrict__ sup_acc) {
    const int lane = threadIdx.x & 31;
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wid >= nsuper * nbr) return;
    const int64_t w = wid / nbr;
    const int k = (int)(wid % nbr);
    int64_t lo = w * T.sup;
    const int64_t hi = min(nchunks, lo + T.sup);
    int64_t acc[3] = {0, 0, 0};
    CsState st;
    uint8_t* src = T.src + (int64_t)(family * nbr + k) * T.nseg;
    CsState* segst = T.segst + (int64_t)(family * nbr + k) * T.nseg;
    if (family == 0) {
        if (w == 0 && (start & CS_EXACT)) {
            // the run's first chunk is the one exact run (candidate 0 started from the true incoming state)
            if (k != 0) {
                if (lane == 0) sup_end[w * nbr + k].freq = sup_end[w * nbr + k].phase = __int_as_float(0x7fc00000);
                return;
            }
            if (lane < P.segs) src[lane] = 0;
            st = ckpt[P.segs];
            lo = 1;
        } else {
            st = ckpt[((int64_t)k * nchunks + lo) * (P.segs + 1)];
        }
    } else {
        const int64_t p = prev_live[w];
        if (p < 0 || (p == 0 && (start & CS_EXACT) && k != 0)) {   // nothing to inherit (family A of super-chunk 0 has one chain only)
            if (lane == 0) sup_end[w * nbr + k].freq = sup_end[w * nbr + k].phase = __int_as_float(0x7fc00000);
            return;
        }
        st = end_a[p * nbr + k];
    }
    st = cs_chain<DT>(iq, n, P, nchunks, nbr, ckpt, nonnoise, chunk_cnt, src, segst, start & CS_CAP, lo, hi, st, acc);
    if (lane == 0) {
        sup_end[w * nbr + k] = st;
        sup_acc[(w * nbr + k) * 3 + 0] = acc[0];
        sup_acc[(w * nbr + k) * 3 + 1] = acc[1];
        sup_acc[(w * nbr + k) * 3 + 2] = acc[2];
    }
}

// prev_live[w] = last super-chunk before w that holds at least one sample above the noise gate (-1: none)
__global__ void k_cs_live(const int* __restrict__ chunk_cnt, int64_t nchunks, int64_t nsuper, int sup, int64_t* __restrict__ live) {
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nsuper) return;
    int64_t any = 0;
    for (int64_t c = w * sup; c < min(nchunks, (w + 1) * (int64_t)sup); c++) any |= chunk_cnt[c] > 0 ? 1 : 0;
    live[w] = any;
}
__global__ void k_cs_prev_live(const int64_t* __restrict__ live, int64_t nsuper, int64_t* __restrict__ prev_live) {
    if (blockIdx.x || threadIdx.x) return;
    int64_t last = -1;
    for (int64_t w = 0; w < nsuper; w++) {
        prev_live[w] = last;
        if (live[w]) last = w;
    }
}

// pass 2b: hop over the super-chunks with the TRUE state.  chosen[w] = table family whose entries are right for super-chunk w
// (k: family A chain k, nbr + k: family B chain k, 2*nbr: the chain this kernel ran itself).
template <int DT>
__global__ void __launch_bounds__(32) k_cs_stitch(const void* __restrict__ iq, int64_t n, CsParams P, int64_t nchunks, int nbr,
                                                  const CsState* __restrict__ ckpt, const int* __restrict__ nonnoise,
                                                  const int* __restrict__ chunk_cnt, CsTables T, int start, int64_t nsuper,
                                                  const int64_t* __restrict__ prev_live, const CsState* __restrict__ end_a,
                                                  const CsState* __restrict__ end_b, const int64_t* __restrict__ acc_a,
                                                  const int64_t* __restrict__ acc_b, uint8_t* __restrict__ chosen,
                                                  int64_t* __restrict__ stats, CsState st_in, CsState* __restrict__ st_out, int hyp_mode,
                                                  int accumulate) {
    // hyp_mode (later shards of a sharded capture): block h hops under the HYPOTHESIS that the shard starts in candidate h's
    // start state (true whenever the preceding shard ends locked); each hypothesis has its own chosen[] row, counters, end
    // state and self-run table, so all of them run concurrently and independently of the preceding shard.
    // accumulate: add the counters to stats[] instead of overwriting them (the ring chunks of a streamed capture sum them).
    const int lane = threadIdx.x;
    const int h = blockIdx.x;
    chosen += (int64_t)h * nsuper;
    if (stats) stats += CS_STATS * h;
    if (st_out) st_out += h;
    const int self_family = 2 * nbr + h;
    int64_t acc[3] = {0, 0, 0};
    int64_t redone = 0, adopted_a = 0, adopted_b = 0;   // super-chunk 0 of the first shard has one chain: not counted
    CsState st = st_in;
    if (hyp_mode) st = ckpt[((int64_t)h * nchunks) * (P.segs + 1)];
    int64_t w = 0;
    if (start & CS_EXACT) {
        if (lane == 0) chosen[0] = 0;
        st = end_a[0];
        for (int q = 0; q < 3; q++) acc[q] += acc_a[q];
        w = 1;
    }
    for (; w < nsuper; w++) {
        const int64_t lo = w * T.sup;
        const int64_t p = prev_live[w];
        // lanes 0..nbr-1: family A start states (candidate checkpoints); lanes 8..8+nbr-1: family B start states
        int m = -1;
        if (lane < nbr) {
            const CsState q = ckpt[((int64_t)lane * nchunks + lo) * (P.segs + 1)];
            if (__float_as_uint(q.freq) == __float_as_uint(st.freq) && __float_as_uint(q.phase) == __float_as_uint(st.phase)) m = lane;
        } else if (lane >= 8 && lane < 8 + nbr && p >= 0) {
            const int k = lane - 8;
            const CsState q = end_a[p * nbr + k];
            const CsState e = end_b[w * nbr + k];
            if (__float_as_uint(q.freq) == __float_as_uint(st.freq) && __float_as_uint(q.phase) == __float_as_uint(st.phase) &&
                e.freq == e.freq)   // NaN end state = chain B k was not run
                m = lane;
        }
        const unsigned any = __ballot_sync(URH_FULL_MASK, m >= 0);
        if (any & 0xffu) {
            const int k = __ffs(any & 0xffu) - 1;
            if (lane == 0) chosen[w] = (uint8_t)k;
            adopted_a++;
            st = end_a[w * nbr + k];
            for (int q = 0; q < 3; q++) acc[q] += acc_a[(w * nbr + k) * 3 + q];
        } else if (any) {
            const int k = __ffs(any) - 1 - 8;
            if (lane == 0) chosen[w] = (uint8_t)(nbr + k);
            adopted_b++;
            st = end_b[w * nbr + k];
            for (int q = 0; q < 3; q++) acc[q] += acc_b[(w * nbr + k) * 3 + q];
        } else {
            if (lane == 0) chosen[w] = (uint8_t)self_family;
            redone++;
            st = cs_chain<DT>(iq, n, P, nchunks, nbr, ckpt, nonnoise, chunk_cnt, T.src + (int64_t)self_family * T.nseg,
                              T.segst + (int64_t)self_family * T.nseg, start & CS_CAP, lo, min(nchunks, lo + T.sup), st, acc);
        }
    }
    if (lane == 0 && st_out) *st_out = st;
    if (lane == 0 && stats) {
        const int64_t v[CS_STATS] = {acc[0], acc[1], acc[2], redone, adopted_a, adopted_b};
        for (int q = 0; q < CS_STATS; q++) stats[q] = (accumulate ? stats[q] : 0) + v[q];
    }
}

// pass 3: out[i] = candidate[src][i] (stepped segments are written by k_cs_fix)
__global__ void k_cs_assemble(const float* __restrict__ cand, int64_t n, CsTables T, int segs, const uint8_t* __restrict__ chosen,
                              float* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t seg = i / CS_SEG;
        const int64_t w = seg / ((int64_t)segs * T.sup);
        const uint8_t k = T.src[(int64_t)chosen[w] * T.nseg + seg];
        if (k != 255) out[i] = cand[(int64_t)k * n + i];
    }
}

// pass 4: the stepped segments (one warp each): recompute the samples from the recorded state
template <int DT>
__global__ void __launch_bounds__(128) k_cs_fix(const void* __restrict__ iq, int64_t n, CsParams P, CsTables T, const uint8_t* __restrict__ chosen,
                                               int cap_start, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t seg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; seg < T.nseg; seg += nw) {
        const int64_t w = seg / ((int64_t)P.segs * T.sup);
        const int64_t t = chosen[w];
        if (T.src[t * T.nseg + seg] != 255) continue;
        CsState st = T.segst[t * T.nseg + seg];
        const int64_t a = seg * CS_SEG;
        for (int g = 0; g < CS_SEG / 32; g++) {
            const int64_t i = a + g * 32 + lane;
            float re = 0.f, im = 0.f;
            bool live = false;
            if (i < n && !(i == 0 && cap_start)) {
                cs_load<DT>(iq, i, re, im);
                live = !(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)) <= P.noise_sqrd);
                if (!live) out[i] = -4.0f;
            } else if (i == 0 && cap_start) {
                out[0] = 0.0f;
            }
            unsigned mask = __ballot_sync(URH_FULL_MASK, live);
            while (mask) {
                const int l = __ffs(mask) - 1;
                mask &= mask - 1;
                const float r1 = __shfl_sync(URH_FULL_MASK, re, l), i1 = __shfl_sync(URH_FULL_MASK, im, l);
                if (lane == 0) {
                    float o;
                    cs_step(st, r1, i1, P, o);
                    out[a + g * 32 + l] = o;
                }
            }
        }
    }
}

int urh_costas_demod_serial(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_sqrd, int loop_order,
                            float bandwidth, float* d_out, const float* d_st_in = nullptr, float* d_st_out = nullptr,
                            int cap_start = 1);  // costas.cu

static int cs_params(urh_ctx* ctx, CsParams* P, int dtype, float noise_sqrd, int order, float bandwidth) {
    const float damping = (float)(sqrt(2.0) / 2.0);
    const double bw = (double)bandwidth, dm = (double)damping;
    volatile float bw2f = bandwidth * bandwidth;
    const double den = (1.0 + ((2.0 * dm) * bw)) + (double)bw2f;
    P->alpha = (float)(((4.0 * dm) * bw) / den);
    P->beta = (float)(((4.0 * bw) * bw) / den);
    P->noise_sqrd = noise_sqrd;
    P->order = order;
    P->segs = 16;
    P->chunk = P->segs * CS_SEG;
    switch (dtype) {
        case URH_DT_I8: P->scale = 127.5f; P->shift = 0.5f; break;
        case URH_DT_U8: P->scale = 127.5f; P->shift = -127.5f; break;
        case URH_DT_I16: P->scale = 32767.5f; P->shift = 0.5f; break;
        case URH_DT_U16: P->scale = 65535.0f; P->shift = -32767.5f; break;
        case URH_DT_F32: P->scale = 1.0f; P->shift = 0.0f; break;
        default: URH_FAIL(ctx, URH_ERR_DTYPE, "Unsupported dtype");
    }
    return URH_OK;
}

struct CsRun {
    CsParams P;
    const void* iq;
    int dtype, nbr, start;   // start: CS_EXACT | CS_CAP
    const CsState* st0 = nullptr;   // exact start: the incoming state on the device (NULL: the loop's initial state)
    int accumulate = 0;             // the stitch adds its counters to stats[] (streamed chunks); cs_finish does not read them
    int64_t n, nchunks;
    float* cand;
    CsState* ckpt;
    int* nonnoise;
    int* chunk_cnt;
    CsTables T;
    int64_t nsuper;
    CsState* sup_end;   // [2][nsuper * nbr]: family A, family B
    int64_t* sup_acc;   // [2][nsuper * nbr * 3]
    int64_t* live;      // [nsuper]
    int64_t* prev_live; // [nsuper]
    uint8_t* chosen;
    int64_t* stats;
    CsState* st_out;
    float* out;
    int adopted;   // hypothesis whose chosen[] row / counters the assemble and fix passes use
};

#define CS_DISPATCH(R, KERNEL, ...)                                                    \
    switch ((R).dtype) {                                                               \
        case URH_DT_I8: URH_LAUNCH(ctx, KERNEL<URH_DT_I8>, __VA_ARGS__); break;        \
        case URH_DT_U8: URH_LAUNCH(ctx, KERNEL<URH_DT_U8>, __VA_ARGS__); break;        \
        case URH_DT_I16: URH_LAUNCH(ctx, KERNEL<URH_DT_I16>, __VA_ARGS__); break;      \
        case URH_DT_U16: URH_LAUNCH(ctx, KERNEL<URH_DT_U16>, __VA_ARGS__); break;      \
        default: URH_LAUNCH(ctx, KERNEL<URH_DT_F32>, __VA_ARGS__); break;              \
    }

// the caller resets the arena (or releases a mark) before: every table below is a fresh arena request
static int cs_speculate(urh_ctx* ctx, CsRun& R) {
    // enough independent chains to fill the GPU: shrink the chunk for short captures (more warm-up overhead)
    int segs = 16;
    while (segs > 2 && (R.n / (segs * CS_SEG)) * R.P.order < (int64_t)ctx->sm_count * 1024) segs >>= 1;
    // $URH_B200_COSTAS_SEGS = 2, 4, 8 or 16 forces the chunk layout (tests run every layout on any capture length); the result
    // does not depend on it
    if (const char* e = getenv("URH_B200_COSTAS_SEGS")) {
        const int f = atoi(e);
        if (f == 2 || f == 4 || f == 8 || f == 16) segs = f;
    }
    R.P.segs = segs;
    R.P.chunk = segs * CS_SEG;
    R.nchunks = urh_div_up(R.n, R.P.chunk);
    R.nbr = R.P.order;  // candidates = lock branches
    URH_CHECK(urh_arena(ctx, (size_t)R.nbr * R.n, &R.cand));
    URH_CHECK(urh_arena(ctx, (size_t)R.nbr * R.nchunks * (R.P.segs + 1), &R.ckpt));
    URH_CHECK(urh_arena(ctx, (size_t)R.nchunks * R.P.segs, &R.nonnoise));
    R.T.nseg = R.nchunks * R.P.segs;
    R.T.sup = (int)max((int64_t)CS_SUP_MIN, urh_div_up((int64_t)131072, (int64_t)R.P.chunk));
    R.nsuper = urh_div_up(R.nchunks, R.T.sup);
    // table families: nbr x A, nbr x B, then one self-run table per stitch hypothesis (a single one when unsharded)
    const int self_tables = (R.start & CS_EXACT) ? 1 : R.nbr;
    URH_CHECK(urh_arena(ctx, (size_t)(2 * R.nbr + self_tables) * R.T.nseg, &R.T.src));
    URH_CHECK(urh_arena(ctx, (size_t)(2 * R.nbr + self_tables) * R.T.nseg, &R.T.segst));
    URH_CHECK(urh_arena(ctx, (size_t)2 * R.nsuper * R.nbr, &R.sup_end));
    URH_CHECK(urh_arena(ctx, (size_t)2 * R.nsuper * R.nbr * 3, &R.sup_acc));
    URH_CHECK(urh_arena(ctx, (size_t)R.nsuper, &R.live));
    URH_CHECK(urh_arena(ctx, (size_t)R.nsuper, &R.prev_live));
    URH_CHECK(urh_arena(ctx, (size_t)R.nsuper * self_tables, &R.chosen));
    URH_CHECK(urh_arena(ctx, (size_t)R.nchunks, &R.chunk_cnt));
    URH_CHECK(urh_arena(ctx, (size_t)CS_STATS * self_tables, &R.stats));
    URH_CHECK(urh_arena(ctx, (size_t)2 * self_tables, &R.st_out));
    R.adopted = 0;
    const dim3 grid((unsigned)urh_div_up(R.nchunks, 128), (unsigned)R.nbr);
    CS_DISPATCH(R, k_cs_speculate, grid, 128, 0, R.iq, R.n, R.P, R.nchunks, R.cand, R.ckpt, R.nonnoise, R.chunk_cnt, R.start, R.st0);
    // pass 2a: the chains of every super-chunk under every assumption (independent of the true incoming state)
    const int64_t per = R.nsuper * R.nbr;
    URH_CUDA(ctx, cudaMemsetAsync(R.sup_acc, 0, (size_t)2 * per * 3 * sizeof(int64_t), ctx->stream));
    URH_LAUNCH(ctx, k_cs_live, (unsigned)urh_div_up(R.nsuper, 128), 128, 0, R.chunk_cnt, R.nchunks, R.nsuper, R.T.sup, R.live);
    URH_LAUNCH(ctx, k_cs_prev_live, 1, 32, 0, (const int64_t*)R.live, R.nsuper, R.prev_live);
    const unsigned gc = (unsigned)urh_div_up(per * 32, 128);
    CS_DISPATCH(R, k_cs_chains, gc, 128, 0, R.iq, R.n, R.P, R.nchunks, R.nbr, R.ckpt, R.nonnoise, R.chunk_cnt, R.T, R.start, R.nsuper, 0,
                (const int64_t*)R.prev_live, (const CsState*)R.sup_end, R.sup_end, R.sup_acc);
    CS_DISPATCH(R, k_cs_chains, gc, 128, 0, R.iq, R.n, R.P, R.nchunks, R.nbr, R.ckpt, R.nonnoise, R.chunk_cnt, R.T, R.start, R.nsuper, 1,
                (const int64_t*)R.prev_live, (const CsState*)R.sup_end, R.sup_end + per, R.sup_acc + per * 3);
    return URH_OK;
}

// assemble + fix with hypothesis R.adopted's chosen[] row; returns that run's end state
static int cs_finish(urh_ctx* ctx, CsRun& R, float* h_state_out) {
    const uint8_t* chosen = R.chosen + (int64_t)R.adopted * R.nsuper;
    const unsigned ga = (unsigned)min(urh_div_up(R.n, 256), (int64_t)ctx->sm_count * 32);
    URH_LAUNCH(ctx, k_cs_assemble, ga, 256, 0, R.cand, R.n, R.T, R.P.segs, chosen, R.out);
    CS_DISPATCH(R, k_cs_fix, (unsigned)min(urh_div_up(R.T.nseg * 32, 128), (int64_t)ctx->sm_count * 16), 128, 0, R.iq, R.n, R.P, R.T, chosen,
                R.start & CS_CAP, R.out);
    if (R.accumulate) return URH_OK;   // streamed: the counters stay on the device until urh_costas_stream_end
    int64_t st6[CS_STATS];
    URH_CHECK(urh_read_i64(ctx, R.stats + CS_STATS * R.adopted, CS_STATS, st6));
    for (int i = 0; i < 3; i++) ctx->costas_stats[i] = st6[i];
    ctx->costas_redone = st6[3];
    ctx->costas_stitch[0] = st6[4];
    ctx->costas_stitch[1] = st6[5];
    ctx->costas_stitch[2] = st6[3];
    ctx->costas_stitch[3] = R.P.segs;
    if (h_state_out) {
        URH_CUDA(ctx, cudaMemcpyAsync(h_state_out, R.st_out + R.adopted, sizeof(CsState), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return URH_OK;
}

static int cs_stitch(urh_ctx* ctx, CsRun& R, CsState st_in, int hypotheses) {
    const int64_t per = R.nsuper * R.nbr;
    CS_DISPATCH(R, k_cs_stitch, hypotheses > 0 ? hypotheses : 1, 32, 0, R.iq, R.n, R.P, R.nchunks, R.nbr, R.ckpt, R.nonnoise, R.chunk_cnt, R.T,
                R.start, R.nsuper, (const int64_t*)R.prev_live, (const CsState*)R.sup_end, (const CsState*)(R.sup_end + per),
                (const int64_t*)R.sup_acc, (const int64_t*)(R.sup_acc + per * 3), R.chosen, R.stats, st_in, R.st_out, hypotheses > 0 ? 1 : 0,
                R.accumulate);
    return URH_OK;
}

static int cs_resolve(urh_ctx* ctx, CsRun& R, CsState st_in, float* h_state_out) {
    URH_CHECK(cs_stitch(ctx, R, st_in, 0));
    R.adopted = 0;
    return cs_finish(ctx, R, h_state_out);
}

int urh_costas_demod(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, float noise_sqrd, int loop_order, float bandwidth,
                     float* d_out) {
    const int order = loop_order > 4 ? 4 : loop_order;  // pyx:285-287
    if (n < 4 * 512 * 4 || (order != 2 && order != 4))
        return urh_costas_demod_serial(ctx, d_iq, dtype, n, noise_sqrd, loop_order, bandwidth, d_out);
    CsRun R;
    URH_CHECK(cs_params(ctx, &R.P, dtype, noise_sqrd, order, bandwidth));
    R.iq = d_iq; R.dtype = dtype; R.n = n; R.start = CS_EXACT | CS_CAP; R.out = d_out;
    urh_arena_reset(ctx);
    URH_CHECK(cs_speculate(ctx, R));
    CsState none;
    none.freq = 0.f; none.phase = 1.5f;
    return cs_resolve(ctx, R, none, nullptr);
}

// Device bytes cs_speculate requests for n samples at loop order `order` (0 for the serial kernel), the largest over the chunk
// layouts: $URH_B200_COSTAS_SEGS may force any of them.  Exact start (one self-run table).  urh_stream_footprint's PSK term.
int64_t urh_costas_arena_bytes(int64_t n, int loop_order) {
    const int order = loop_order > 4 ? 4 : loop_order;
    if (n < 4 * 512 * 4 || (order != 2 && order != 4)) return 0;
    auto r = [](int64_t b) { return b > 0 ? (b + 255) & ~(int64_t)255 : (int64_t)256; };
    int64_t most = 0;
    for (int segs = 2; segs <= CS_MAX_SEGS; segs <<= 1) {
        const int64_t chunk = (int64_t)segs * CS_SEG, nchunks = urh_div_up(n, chunk), nseg = nchunks * segs;
        const int64_t sup = max((int64_t)CS_SUP_MIN, urh_div_up((int64_t)131072, chunk)), nsuper = urh_div_up(nchunks, sup);
        const int64_t nbr = order, fam = 2 * nbr + 1;
        const int64_t b = r(nbr * n * 4) + r(nbr * nchunks * (segs + 1) * (int64_t)sizeof(CsState)) + r(nseg * 4) + r(fam * nseg) +
                          r(fam * nseg * (int64_t)sizeof(CsState)) + r(2 * nsuper * nbr * (int64_t)sizeof(CsState)) +
                          r(2 * nsuper * nbr * 3 * 8) + 2 * r(nsuper * 8) + r(nsuper) + r(nchunks * 4) + r(CS_STATS * 8) +
                          r(2 * (int64_t)sizeof(CsState));
        most = b > most ? b : most;
    }
    return most;
}

// ---- PSK captures streamed through a ring of device slots (digitize.cu, DESIGN.md §4.3) --------------------------------------------
// The ring chunks run one after the other on the compute stream, so the exact loop state at every chunk edge is on the device when
// the next chunk starts: chunk c > 0 is an exact start (no capture start), its incoming state the one chunk c - 1 left.  Chunk c reads
// state slot c & 1 and writes slot (c + 1) & 1.  The stitch counters add up in S->acc; nothing is read back per chunk.
__global__ void k_cs_stream_init(CsState* st, int64_t* acc) {
    if (threadIdx.x == 0) {
        st[0].freq = 0.0f;
        st[0].phase = 1.5f;
    }
    if (threadIdx.x < CS_STATS) acc[threadIdx.x] = 0;
}

int urh_costas_stream_begin(urh_ctx* ctx, UrhCostasStream* S) {
    CsState* st;
    URH_CHECK(urh_arena(ctx, 2, &st));
    URH_CHECK(urh_arena(ctx, CS_STATS, &S->acc));
    S->state = (float*)st;
    S->segs = 0;
    URH_LAUNCH(ctx, k_cs_stream_init, 1, 32, 0, st, S->acc);
    return URH_OK;
}

// ring chunk c: n samples at d_iq (the chunk's first sample at index 0) -> d_out[n]; enqueued only
int urh_costas_stream_chunk(urh_ctx* ctx, UrhCostasStream* S, int64_t c, const void* d_iq, int dtype, int64_t n, float noise_sqrd,
                            int loop_order, float bandwidth, float* d_out) {
    CsState* st = (CsState*)S->state;
    CsState* st_in = st + (c & 1);
    CsState* st_out = st + ((c + 1) & 1);
    const int order = loop_order > 4 ? 4 : loop_order;
    if (n < 4 * 512 * 4 || (order != 2 && order != 4))
        return urh_costas_demod_serial(ctx, d_iq, dtype, n, noise_sqrd, loop_order, bandwidth, d_out, (const float*)st_in, (float*)st_out,
                                       c == 0);
    CsRun R;
    URH_CHECK(cs_params(ctx, &R.P, dtype, noise_sqrd, order, bandwidth));
    R.iq = d_iq; R.dtype = dtype; R.n = n; R.start = CS_EXACT | (c == 0 ? CS_CAP : 0); R.st0 = st_in; R.out = d_out;
    URH_CHECK(cs_speculate(ctx, R));
    R.stats = S->acc;
    R.st_out = st_out;
    R.accumulate = 1;
    if (S->segs == 0) S->segs = R.P.segs;
    CsState none;
    none.freq = 0.f; none.phase = 1.5f;   // unused: an exact start takes its state from st0
    URH_CHECK(cs_stitch(ctx, R, none, 0));
    R.adopted = 0;
    return cs_finish(ctx, R, nullptr);
}

// after the last chunk: the summed counters become urh_costas_stats / urh_costas_stitch_stats (one read-back per call)
int urh_costas_stream_end(urh_ctx* ctx, const UrhCostasStream* S) {
    int64_t st6[CS_STATS];
    URH_CHECK(urh_read_i64(ctx, S->acc, CS_STATS, st6));
    for (int i = 0; i < 3; i++) ctx->costas_stats[i] = st6[i];
    ctx->costas_redone = st6[3];
    ctx->costas_stitch[0] = st6[4];
    ctx->costas_stitch[1] = st6[5];
    ctx->costas_stitch[2] = st6[3];
    ctx->costas_stitch[3] = S->segs;
    return URH_OK;
}

// ---- PSK captures sharded over GPUs: pass 1 runs concurrently on every rank, the chain is handed from rank to rank ----
// d_iq points at the shard's first own sample; later shards have URH_COSTAS_HALO samples of the preceding shard stored in
// front of it.  urh_costas_shard_speculate is asynchronous; urh_costas_shard_resolve needs the preceding shard's final
// loop state (state_in = {freq, phase}; ignored on the first shard) and returns this shard's.
// The run lives on the context, so every context of a process can hold its own sharded run between these calls.
static CsRun& shard_run(urh_ctx* ctx) {
    if (!ctx->costas_shard) ctx->costas_shard = new CsRun();
    return *(CsRun*)ctx->costas_shard;
}

void urh_costas_shard_release(urh_ctx* ctx) {
    delete (CsRun*)ctx->costas_shard;
    ctx->costas_shard = nullptr;
}

extern "C" int urh_costas_halo_samples(void) { return CS_WARM; }

extern "C" int urh_costas_shard_speculate(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, int first_shard, float noise_mag,
                                          int loop_order, float bandwidth, float* d_out) {
    const int order = loop_order > 4 ? 4 : loop_order;
    if (order != 2 && order != 4) URH_FAIL(ctx, URH_ERR_INVALID, "sharded PSK: loop order 2 or 4");
    volatile float nm = noise_mag;
    volatile float sq = nm * nm;
    CsRun& R = shard_run(ctx);
    URH_CHECK(cs_params(ctx, &R.P, dtype, sq, order, bandwidth));
    R.iq = d_iq; R.dtype = dtype; R.n = n; R.start = first_shard ? (CS_EXACT | CS_CAP) : 0; R.out = d_out;
    R.st0 = nullptr;
    R.accumulate = 0;
    urh_arena_reset(ctx);
    return cs_speculate(ctx, R);
}

extern "C" int urh_costas_shard_resolve(urh_ctx* ctx, const float* h_state_in, float* h_state_out) {
    CsState in;
    in.freq = h_state_in ? h_state_in[0] : 0.f;
    in.phase = h_state_in ? h_state_in[1] : 1.5f;
    return cs_resolve(ctx, shard_run(ctx), in, h_state_out);
}

// Later shards: hop over the shard under each of the `order` hypotheses "the shard starts in candidate h's start state",
// all at once (one warp each), independent of the preceding shard.  h_out[h] = {start.freq, start.phase, end.freq, end.phase}.
// The first shard has one true run: h_out[0] = {initial state, end state}.  Returns the number of hypotheses in *count.
extern "C" int urh_costas_shard_hypotheses(urh_ctx* ctx, float* h_out, int* count) {
    CsRun& R = shard_run(ctx);
    const bool first_shard = R.start & CS_EXACT;
    const int nh = first_shard ? 1 : R.nbr;
    CsState none;
    none.freq = 0.f; none.phase = 1.5f;
    URH_CHECK(cs_stitch(ctx, R, none, first_shard ? 0 : nh));
    CsState ends[4], starts[4];
    URH_CUDA(ctx, cudaMemcpyAsync(ends, R.st_out, sizeof(CsState) * nh, cudaMemcpyDeviceToHost, ctx->stream));
    for (int h = 0; h < nh && !first_shard; h++)
        URH_CUDA(ctx, cudaMemcpyAsync(&starts[h], R.ckpt + ((int64_t)h * R.nchunks) * (R.P.segs + 1), sizeof(CsState), cudaMemcpyDeviceToHost, ctx->stream));
    URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (first_shard) starts[0] = none;
    for (int h = 0; h < nh; h++) {
        h_out[4 * h + 0] = starts[h].freq; h_out[4 * h + 1] = starts[h].phase;
        h_out[4 * h + 2] = ends[h].freq; h_out[4 * h + 3] = ends[h].phase;
    }
    *count = nh;
    return URH_OK;
}

// Adopt hypothesis h (its start state equalled, bit for bit, the preceding shard's end state): assemble + fix.
extern "C" int urh_costas_shard_adopt(urh_ctx* ctx, int h, float* h_state_out) {
    CsRun& R = shard_run(ctx);
    if (h < 0 || h >= ((R.start & CS_EXACT) ? 1 : R.nbr)) URH_FAIL(ctx, URH_ERR_INVALID, "costas_shard_adopt: no such hypothesis");
    R.adopted = h;
    return cs_finish(ctx, R, h_state_out);
}

// diagnostics of the last speculative run: {chunks resolved in O(1), chunks walked, samples stepped serially}
extern "C" int urh_costas_stats(urh_ctx* ctx, int64_t* h_out3) {
    for (int i = 0; i < 3; i++) h_out3[i] = ctx->costas_stats[i];
    return URH_OK;
}

// super-chunks whose chain the stitch pass had to run itself in the last speculative run (no assumption matched)
extern "C" int64_t urh_costas_last_redone(urh_ctx* ctx) { return ctx->costas_redone; }

// how the stitch pass of the last PSK demodulation resolved its super-chunks: {adopted from family A, adopted from family B,
// chained by the stitch warp itself, segs}.  Super-chunk 0 of an unsharded capture (or of the first shard) is not counted: it
// has one chain only.  The serial kernel reports {0, 0, 0, 0}.
extern "C" int urh_costas_stitch_stats(urh_ctx* ctx, int64_t* h_out4) {
    for (int i = 0; i < 4; i++) h_out4[i] = ctx->costas_stitch[i];
    return URH_OK;
}
