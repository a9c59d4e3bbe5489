// IQArray.export_to_sub (IQArray.py:275-319): the Flipper Zero RAW_Data body of a capture, generated on the device.
//
// The reference walks u = convert_to(uint8)[:, 0] sample by sample with (lastvalue, counter).  Restated over the runs of equal
// values (DESIGN §4.12), the walk is a machine over runs with 257 states: A ("armed at the next run's first sample") and S_v
// ("armed on value v by a run of one sample, skipping to the next run of v").  A run of length >= 2 met in A emits its length
// and stays in A; a run of one sample met in A goes to S_v; a run of v met in S_v emits 1 + its length and goes to A; every
// other run leaves S_v as it is.  The walk starts in A at sample 0; ending in S_v emits 1.
//
// A tile owns the runs that START in it.  Its transition function (257 entries) is found in shared memory by pointer doubling
// over the in-tile successors of its runs (k_sub_tiles); the tiles' entry states come from a grouped prefix composition of
// those tables (k_sub_compose / k_sub_down); the emitted entries are the runs on the chain, marked by doubling again, their
// byte lengths summed by the look-back scan and the decimal text written in place (k_sub_text).  No pass walks the capture,
// the tiles or the runs on one thread.
#include <errno.h>
#include <unistd.h>

#include "convert.cuh"
#include "stream_ring.cuh"
#include "tilescan.cuh"

namespace {

constexpr int SUB_T = 2048;                       // samples per tile
constexpr int SUB_THREADS = 256;
constexpr int SUB_PER = SUB_T / SUB_THREADS;      // samples (and run slots) per thread
constexpr int SUB_CHUNKS = SUB_T / 32;            // 32-run chunks of a tile's run list
constexpr int SUB_STATES = 257;                   // S_0 .. S_255, then A
constexpr uint16_t SUB_A = 256;
constexpr uint16_t SUB_NONE = 0xFFFF;
constexpr uint16_t SUB_LONG = 0x8000;             // pos[k] flag: run k has at least 2 samples
constexpr int SUB_G = 32;                         // tables composed per block
constexpr int SUB_LINE = 512;                     // entries per RAW_Data line

struct SubCnt {
    int64_t e, b;   // entries, bytes without the 10 extra bytes of each line's "RAW_Data: "
};
struct AddCnt {
    __device__ __forceinline__ SubCnt operator()(SubCnt a, SubCnt b) const { return SubCnt{a.e + b.e, a.b + b.b}; }
};
struct MinI64 {
    __device__ __forceinline__ int64_t operator()(int64_t a, int64_t b) const { return a < b ? a : b; }
};

// one tile's runs in shared memory; `occ` (the per-chunk next-occurrence table) is dead once ns[] is known and its space holds
// the doubling buffers
struct SubTile {
    uint8_t u[SUB_T + 2];          // samples t0 - 1 .. t0 + SUB_T (the halos where they exist)
    uint16_t pos[SUB_T];           // tile-local first sample of run k | SUB_LONG
    uint8_t val[SUB_T];
    uint16_t ns[SUB_T];            // the next run of the same value in the tile (SUB_NONE: none)
    uint16_t first[256];           // the first run of each value in the tile
    union alignas(16) {
        uint16_t occ[SUB_CHUNKS + 1][256];
        struct {
            uint16_t j[2][SUB_T + 1];
            uint8_t mark[SUB_T + 1];
        } w;
    };
    int warp_sum[SUB_THREADS / 32];
    int R;
};

template <typename S>
struct SubFromIQ {   // column I of the capture, as convert_to(uint8) gives it
    const S* iq;
    __device__ __forceinline__ uint8_t operator()(int64_t i) const { return conv_one<S, uint8_t>(iq[2 * i]); }
};
template <>
struct SubFromIQ<uint8_t> {
    const uint8_t* iq;
    __device__ __forceinline__ uint8_t operator()(int64_t i) const { return iq[2 * i]; }
};
struct SubFromCol {   // the uint8 column k_sub_tiles left behind
    const uint8_t* col;
    __device__ __forceinline__ uint8_t operator()(int64_t i) const { return col[i]; }
};

__device__ __forceinline__ int sub_block_excl_sum(SubTile& s, int x, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(URH_FULL_MASK, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s.warp_sum[warp] = incl;
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < SUB_THREADS / 32; w++) {
        before += (w < warp) ? s.warp_sum[w] : 0;
        all += s.warp_sum[w];
    }
    __syncthreads();
    *total = all;
    return before + incl - x;
}

// Loads the tile's samples, lists the runs starting in it, finds every run's next run of the same value (warp match inside a
// 32-run chunk, a suffix table of first occurrences across chunks) and leaves the in-tile successor of every run in w.j[0]:
// the run armed after it, R for "the first run of a later tile" (A), R + 1 + v for "still skipping on v" (S_v).
template <typename Get>
__device__ void sub_build(SubTile& s, Get get, int64_t n, int64_t t0, int cnt, uint8_t* col) {
    const int tid = threadIdx.x, lane = tid & 31;
    for (int j = tid; j < cnt + 2; j += SUB_THREADS) {
        const int64_t i = t0 - 1 + j;
        if (i >= 0 && i < n) {
            const uint8_t v = get(i);
            s.u[j] = v;
            if (col && j >= 1 && j <= cnt) col[i] = v;
        }
    }
    __syncthreads();
    const int j0 = tid * SUB_PER;
    int starts = 0;
#pragma unroll
    for (int q = 0; q < SUB_PER; q++) {
        const int j = j0 + q;
        starts += (j < cnt && (t0 + j == 0 || s.u[j + 1] != s.u[j])) ? 1 : 0;
    }
    int R;
    int k = sub_block_excl_sum(s, starts, &R);
#pragma unroll
    for (int q = 0; q < SUB_PER; q++) {
        const int j = j0 + q;
        if (j < cnt && (t0 + j == 0 || s.u[j + 1] != s.u[j])) {
            const bool is_long = t0 + j + 1 < n && s.u[j + 2] == s.u[j + 1];
            s.pos[k] = (uint16_t)(j | (is_long ? SUB_LONG : 0));
            s.val[k] = s.u[j + 1];
            k++;
        }
    }
    const int nch = (R + 31) >> 5;
    uint32_t* occ32 = (uint32_t*)&s.occ[0][0];
    for (int i = tid; i < (nch + 1) * 128; i += SUB_THREADS) occ32[i] = 0xFFFFFFFFu;
    if (tid == 0) s.R = R;
    __syncthreads();
    for (int r = tid; r < nch * 32; r += SUB_THREADS) {   // whole warps: nch * 32 and SUB_THREADS are multiples of 32
        const int v = r < R ? (int)s.val[r] : 256 + lane;
        const uint32_t m = __match_any_sync(URH_FULL_MASK, v);
        if (r < R) {
            if (__ffs(m) - 1 == lane) s.occ[r >> 5][v] = (uint16_t)r;
            const uint32_t later = m & ~((2u << lane) - 1u);
            s.ns[r] = later ? (uint16_t)(r - lane + __ffs(later) - 1) : SUB_NONE;
        }
    }
    __syncthreads();
    {   // occ[c][v] <- the first run of v in chunks >= c (tid = v)
        uint16_t cur = SUB_NONE;
        for (int c = nch - 1; c >= 0; c--) {
            const uint16_t x = s.occ[c][tid];
            if (x != SUB_NONE) cur = x;
            s.occ[c][tid] = cur;
        }
        s.first[tid] = cur;
    }
    __syncthreads();
    for (int r = tid; r < R; r += SUB_THREADS)
        if (s.ns[r] == SUB_NONE) s.ns[r] = s.occ[(r >> 5) + 1][s.val[r]];
    __syncthreads();
    for (int r = tid; r <= R; r += SUB_THREADS) {
        uint16_t nx = (uint16_t)R;
        if (r < R) {
            if (s.pos[r] & SUB_LONG) nx = (uint16_t)(r + 1);
            else if (s.ns[r] != SUB_NONE) nx = (uint16_t)(s.ns[r] + 1);
            else nx = (uint16_t)(R + 1 + s.val[r]);
        }
        s.w.j[0][r] = nx;
    }
    __syncthreads();
}

// Pass 1: the uint8 column, the tile's transition table and its first run start (n: none).
template <typename Get>
__global__ void __launch_bounds__(SUB_THREADS) k_sub_tiles(Get get, int64_t n, uint8_t* __restrict__ col, uint16_t* __restrict__ fn,
                                                           int64_t* __restrict__ first_start) {
    __shared__ SubTile s;
    const int64_t t = blockIdx.x, t0 = t * SUB_T;
    const int cnt = (int)min((int64_t)SUB_T, n - t0);
    sub_build(s, get, n, t0, cnt, col);
    const int R = s.R;
    int b = 0;
    for (int step = 1; step <= R; step <<= 1) {   // j[b] = successor^(2^r): after the loop, every run's exit node
        for (int r = threadIdx.x; r <= R; r += SUB_THREADS) {
            const uint16_t x = s.w.j[b][r];
            s.w.j[b ^ 1][r] = x < R ? s.w.j[b][x] : x;
        }
        __syncthreads();
        b ^= 1;
    }
    auto state = [&](int node) -> uint16_t {
        const int x = s.w.j[b][node];
        return x == R ? SUB_A : (uint16_t)(x - R - 1);
    };
    uint16_t* f = fn + t * SUB_STATES;
    const int v = threadIdx.x;
    f[v] = s.first[v] == SUB_NONE ? (uint16_t)v : state(s.first[v] + 1);
    if (v == 0) {
        f[SUB_A] = state(0);
        first_start[t] = R ? t0 + (s.pos[0] & ~SUB_LONG) : n;
    }
}

// In-place inclusive prefix composition of the tables of each group of SUB_G tiles: tab[i][s] <- state after tiles g0..i from s.
// up[g] receives the group's whole function.
__global__ void __launch_bounds__(288) k_sub_compose(uint16_t* __restrict__ tab, int64_t m, uint16_t* __restrict__ up) {
    const int s = threadIdx.x;
    const int64_t g0 = (int64_t)blockIdx.x * SUB_G;
    const int cnt = (int)min((int64_t)SUB_G, m - g0);
    uint16_t xs[SUB_G];
    uint16_t x = (uint16_t)s;
    if (s < SUB_STATES) {
#pragma unroll
        for (int i = 0; i < SUB_G; i++) {
            if (i < cnt) x = __ldcg(tab + (g0 + i) * SUB_STATES + x);
            xs[i] = x;
        }
    }
    __syncthreads();
    if (s < SUB_STATES) {
#pragma unroll
        for (int i = 0; i < SUB_G; i++)
            if (i < cnt) tab[(g0 + i) * SUB_STATES + s] = xs[i];
        up[(int64_t)blockIdx.x * SUB_STATES + s] = x;
    }
}

// Entry states of the elements of one level from their groups' entry states (e_up == NULL: the one group enters in A).
// count = m + 1 at the bottom level: entry[m] is the state after the last tile.
__global__ void k_sub_down(const uint16_t* __restrict__ tab, int64_t m, const uint16_t* __restrict__ e_up, uint16_t* __restrict__ e,
                           int64_t count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (i < m && i % SUB_G == 0) {
        e[i] = e_up ? e_up[i / SUB_G] : SUB_A;
        return;
    }
    const uint16_t pe = e_up ? e_up[(i - 1) / SUB_G] : SUB_A;
    e[i] = tab[(i - 1) * SUB_STATES + pe];
}

struct SubNextStart {   // next[t] = first run start in tiles > t (n: none), a suffix minimum read backwards
    const int64_t* first;
    int64_t* next;
    int64_t nt;
    __device__ __forceinline__ int64_t load(int64_t i) const { return first[nt - 1 - i]; }
    __device__ __forceinline__ void post(int64_t i, int64_t excl, int64_t) const { next[nt - 1 - i] = excl; }
};
struct SubOffsets {
    SubCnt* cnt;
    __device__ __forceinline__ SubCnt load(int64_t i) const { return cnt[i]; }
    __device__ __forceinline__ void post(int64_t i, SubCnt excl, SubCnt) const { cnt[i] = excl; }
};

__device__ __forceinline__ int sub_digits(int64_t c) {
    int d = 1;
    while (c >= 10) {
        c /= 10;
        d++;
    }
    return d;
}
__device__ __forceinline__ int64_t sub_bytes(int64_t c, int v) { return 1 + (v <= 127 ? 1 : 0) + sub_digits(c); }

// entry idx (0-based over the file) at byte `at` of the body: "\nRAW_Data: " or " ", the sign, the digits
__device__ __forceinline__ void sub_put(uint8_t* out, int64_t cap, int64_t idx, int64_t at, int64_t c, int v) {
    if (at + 32 > cap) return;   // never past the buffer (the call fails on a length above the bound)
    uint8_t* p = out + at;
    if (idx % SUB_LINE == 0) {
        const char* pre = "\nRAW_Data: ";
#pragma unroll
        for (int q = 0; q < 11; q++) p[q] = (uint8_t)pre[q];
        p += 11;
    } else {
        *p++ = ' ';
    }
    if (v <= 127) *p++ = '-';
    const int d = sub_digits(c);
    for (int q = d - 1; q >= 0; q--) {
        p[q] = (uint8_t)('0' + c % 10);
        c /= 10;
    }
}

// Passes 2 and 3: the entries this tile emits, given its entry state.  WRITE = 0 stores their count and byte sum in cnt[t];
// WRITE = 1 reads the exclusive prefix from there and writes their text; tile t = t_begin + block, byte b of the body at out[b - base].
template <int WRITE>
__global__ void __launch_bounds__(SUB_THREADS) k_sub_text(const uint8_t* __restrict__ col, int64_t n, const uint16_t* __restrict__ entry,
                                                          int64_t nt, const int64_t* __restrict__ next_start, SubCnt* __restrict__ cnt,
                                                          uint8_t* __restrict__ out, int64_t cap, int64_t t_begin, int64_t base) {
    __shared__ SubTile s;
    const int64_t t = t_begin + blockIdx.x, t0 = t * SUB_T;
    const int c = (int)min((int64_t)SUB_T, n - t0);
    sub_build(s, SubFromCol{col}, n, t0, c, nullptr);
    const int R = s.R, tid = threadIdx.x;
    const int64_t end_local = next_start[t] - t0;   // end of the tile's last run
    auto run_len = [&](int k) -> int64_t {
        const int64_t e = k + 1 < R ? (int64_t)(s.pos[k + 1] & ~SUB_LONG) : end_local;
        return e - (s.pos[k] & ~SUB_LONG);
    };
    const uint16_t e_in = entry[t];
    // the chain's first armed run: 0 in A; after the first run of v in S_v (which emits), none if v does not start a run here
    int c0 = R;
    int pre_v = -1;
    int64_t pre_c = 0;
    if (e_in == SUB_A) {
        c0 = 0;
    } else if (s.first[e_in] != SUB_NONE) {
        pre_v = e_in;
        pre_c = 1 + run_len(s.first[e_in]);
        c0 = s.first[e_in] + 1;
    }
    for (int r = tid; r <= R; r += SUB_THREADS) s.w.mark[r] = r == c0;
    __syncthreads();
    int b = 0;
    for (int step = 1; step <= R; step <<= 1) {   // after round r every run succ^i(c0), i < 2^(r+1), is marked
        for (int r = tid; r <= R; r += SUB_THREADS) {
            const uint16_t x = s.w.j[b][r];
            if (r < R && s.w.mark[r] && x < R) s.w.mark[x] = 1;
            s.w.j[b ^ 1][r] = x < R ? s.w.j[b][x] : x;
        }
        __syncthreads();
        b ^= 1;
    }
    // thread tid emits for runs [tid * SUB_PER, +SUB_PER) in order; thread 0 first emits the entry state's, the last thread of
    // the last tile the final one of a walk that ends skipping
    const int fin_v = (t == nt - 1 && entry[nt] != SUB_A) ? entry[nt] : -1;
    auto emission = [&](int k, int64_t& cc, int& v) -> bool {
        if (k >= R || !s.w.mark[k]) return false;
        v = s.val[k];
        if (s.pos[k] & SUB_LONG) cc = run_len(k);
        else if (s.ns[k] != SUB_NONE) cc = 1 + run_len(s.ns[k]);
        else return false;
        return true;
    };
    int my_e = 0;
    int64_t my_b = 0;
    if (tid == 0 && pre_v >= 0) {
        my_e++;
        my_b += sub_bytes(pre_c, pre_v);
    }
    for (int q = 0; q < SUB_PER; q++) {
        int64_t cc;
        int v;
        if (emission(tid * SUB_PER + q, cc, v)) {
            my_e++;
            my_b += sub_bytes(cc, v);
        }
    }
    if (tid == SUB_THREADS - 1 && fin_v >= 0) {
        my_e++;
        my_b += sub_bytes(1, fin_v);
    }
    // block exclusive scan of (entries, bytes): entries through the int helper, bytes through a second pass of the same
    int tot_e;
    const int ex_e = sub_block_excl_sum(s, my_e, &tot_e);
    __shared__ long long s_wb[SUB_THREADS / 32];
    long long incl = my_b;
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(URH_FULL_MASK, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_wb[warp] = incl;
    __syncthreads();
    long long ex_b = incl - my_b, tot_b = 0;
#pragma unroll
    for (int w = 0; w < SUB_THREADS / 32; w++) {
        ex_b += (w < warp) ? s_wb[w] : 0;
        tot_b += s_wb[w];
    }
    if (!WRITE) {
        if (tid == 0) cnt[t] = SubCnt{tot_e, tot_b};
        return;
    }
    const SubCnt off = cnt[t];
    int64_t idx = off.e + ex_e, at = off.b + ex_b;
    auto put = [&](int64_t cc, int v) {
        sub_put(out, cap, idx, at + 10 * ((idx + SUB_LINE - 1) / SUB_LINE) - base, cc, v);
        at += sub_bytes(cc, v);
        idx++;
    };
    if (tid == 0 && pre_v >= 0) put(pre_c, pre_v);
    for (int q = 0; q < SUB_PER; q++) {
        int64_t cc;
        int v;
        if (emission(tid * SUB_PER + q, cc, v)) put(cc, v);
    }
    if (tid == SUB_THREADS - 1 && fin_v >= 0) put(1, fin_v);
}

template <typename S>
__global__ void k_sub_column(const S* __restrict__ iq, int64_t count, uint8_t* __restrict__ col) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) col[i] = SubFromIQ<S>{iq}(i);
}

// the most body bytes n samples give: every entry but the last covers at least 2 samples at most 1.5 bytes each ("-2 "); 32 of
// the 48 spare bytes let the writer check a whole entry against the buffer's end
static int64_t urh_sub_export_bound_(int64_t n) {
    if (n <= 0) return 0;
    return (3 * n + 3) / 2 + 10 * ((n / 2 + 1 + SUB_LINE - 1) / SUB_LINE) + 48;
}

// The device scratch of one export: the uint8 column, the table levels (m_0 = nt tiles, m_{l+1} = ceil(m_l / SUB_G) until one group
// is left), the entry states of every composed level, the first / next run starts and the (entries, bytes) table of the tiles.
struct SubPlan {
    int64_t n = 0, nt = 0;
    std::vector<int64_t> m;
    int L = 0;
    std::vector<uint16_t*> tab, ent;
    uint8_t* col = nullptr;
    int64_t *first = nullptr, *next = nullptr;
    SubCnt *cnt = nullptr, *total = nullptr;
    // arena bytes of the requests above (urh_arena_alloc rounds each to 256)
    int64_t bytes() const {
        int64_t b = r256(n) + 2 * r256(nt * 8) + r256(nt * (int64_t)sizeof(SubCnt)) + 256;
        for (int l = 0; l <= L; l++) b += r256(m[l] * SUB_STATES * 2);
        for (int l = 0; l < L; l++) b += r256((m[l] + 1) * 2);
        return b;
    }
};

static void sub_levels(SubPlan& P, int64_t n) {
    P.n = n;
    P.nt = urh_div_up(n, SUB_T);
    P.m.assign(1, P.nt);
    while (P.m.back() > 1 || P.m.size() == 1) P.m.push_back(urh_div_up(P.m.back(), SUB_G));
    P.L = (int)P.m.size() - 1;   // composed levels 0 .. L-1; level L has one element
}

static int sub_plan(urh_ctx* ctx, SubPlan& P, int64_t n) {
    sub_levels(P, n);
    P.tab.resize(P.L + 1);
    P.ent.resize(P.L);
    URH_CHECK(urh_arena(ctx, (size_t)n, &P.col));
    for (int l = 0; l <= P.L; l++) URH_CHECK(urh_arena(ctx, (size_t)P.m[l] * SUB_STATES, &P.tab[l]));
    for (int l = 0; l < P.L; l++) URH_CHECK(urh_arena(ctx, (size_t)P.m[l] + 1, &P.ent[l]));
    URH_CHECK(urh_arena(ctx, (size_t)P.nt, &P.first));
    URH_CHECK(urh_arena(ctx, (size_t)P.nt, &P.next));
    URH_CHECK(urh_arena(ctx, (size_t)P.nt, &P.cnt));
    URH_CHECK(urh_arena(ctx, 1, &P.total));
    return URH_OK;
}

// Pass 1 over the capture (col filled) or over a column already on the device (d_iq NULL)
static int sub_tiles(urh_ctx* ctx, const SubPlan& P, const void* d_iq, int dtype) {
    const unsigned g = (unsigned)P.nt;
    if (!d_iq) {
        URH_LAUNCH(ctx, k_sub_tiles<SubFromCol>, g, SUB_THREADS, 0, SubFromCol{P.col}, P.n, (uint8_t*)nullptr, P.tab[0], P.first);
        return URH_OK;
    }
    switch (dtype) {
        case URH_DT_I8: URH_LAUNCH(ctx, k_sub_tiles<SubFromIQ<int8_t>>, g, SUB_THREADS, 0, SubFromIQ<int8_t>{(const int8_t*)d_iq}, P.n, P.col, P.tab[0], P.first); break;
        case URH_DT_U8: URH_LAUNCH(ctx, k_sub_tiles<SubFromIQ<uint8_t>>, g, SUB_THREADS, 0, SubFromIQ<uint8_t>{(const uint8_t*)d_iq}, P.n, P.col, P.tab[0], P.first); break;
        case URH_DT_I16: URH_LAUNCH(ctx, k_sub_tiles<SubFromIQ<int16_t>>, g, SUB_THREADS, 0, SubFromIQ<int16_t>{(const int16_t*)d_iq}, P.n, P.col, P.tab[0], P.first); break;
        case URH_DT_U16: URH_LAUNCH(ctx, k_sub_tiles<SubFromIQ<uint16_t>>, g, SUB_THREADS, 0, SubFromIQ<uint16_t>{(const uint16_t*)d_iq}, P.n, P.col, P.tab[0], P.first); break;
        default: URH_LAUNCH(ctx, k_sub_tiles<SubFromIQ<float>>, g, SUB_THREADS, 0, SubFromIQ<float>{(const float*)d_iq}, P.n, P.col, P.tab[0], P.first); break;
    }
    return URH_OK;
}

// After pass 1: entry states, next run starts, the count pass and the offsets scan (cnt[t] <- exclusive (entries, bytes))
static int sub_chain(urh_ctx* ctx, const SubPlan& P) {
    for (int l = 0; l < P.L; l++) URH_LAUNCH(ctx, k_sub_compose, (unsigned)P.m[l + 1], 288, 0, P.tab[l], P.m[l], P.tab[l + 1]);
    for (int l = P.L - 1; l >= 0; l--) {
        const int64_t count = P.m[l] + (l == 0 ? 1 : 0);
        URH_LAUNCH(ctx, k_sub_down, (unsigned)urh_div_up(count, 256), 256, 0, P.tab[l], P.m[l], l + 1 < P.L ? P.ent[l + 1] : nullptr,
                   P.ent[l], count);
    }
    URH_CHECK(urhts::scan(ctx, P.nt, P.n, MinI64{}, SubNextStart{P.first, P.next, P.nt}, (int64_t*)nullptr));
    URH_LAUNCH(ctx, k_sub_text<0>, (unsigned)P.nt, SUB_THREADS, 0, P.col, P.n, P.ent[0], P.nt, P.next, P.cnt, (uint8_t*)nullptr,
               (int64_t)0, (int64_t)0, (int64_t)0);
    URH_CHECK(urhts::scan(ctx, P.nt, SubCnt{0, 0}, AddCnt{}, SubOffsets{P.cnt}, P.total));
    return URH_OK;
}

// body byte offset of tile t (t == nt: the body's length); synchronises
static int sub_offset(urh_ctx* ctx, const SubPlan& P, int64_t t, int64_t* at) {
    int64_t h[2];
    URH_CHECK(urh_read_i64(ctx, (const int64_t*)(t < P.nt ? P.cnt + t : P.total), 2, h));
    *at = h[1] + 10 * ((h[0] + SUB_LINE - 1) / SUB_LINE);
    return URH_OK;
}

// text tiles per piece of a streamed body: the chunk's whole tiles
static int64_t sub_piece_tiles(int64_t n, int64_t chunk_samples) { return stream_chunk_samples(n, chunk_samples) / SUB_T; }
static int64_t sub_piece_cap(int64_t n, int64_t chunk_samples) {
    return r256(urh_sub_export_bound_(sub_piece_tiles(n, chunk_samples) * SUB_T) + 128);
}

}  // namespace

extern "C" int64_t urh_sub_export_bound(int64_t n) { return urh_sub_export_bound_(n); }

extern "C" int urh_sub_export(urh_ctx* ctx, const void* d_iq, int dtype, int64_t n, uint8_t* d_out, int64_t capacity, int64_t* h_bytes) {
    if (!d_iq || !d_out || !h_bytes || n <= 0) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: bad arguments");
    if (urh_iq_bytes(dtype) == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Data type not supported");
    if (capacity < urh_sub_export_bound(n)) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: output buffer below urh_sub_export_bound");
    if (urh_div_up(n, SUB_T) >= (1ll << 31)) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: capture too long");
    urh_arena_reset(ctx);
    SubPlan P;
    URH_CHECK(sub_plan(ctx, P, n));
    URH_CHECK(sub_tiles(ctx, P, d_iq, dtype));
    URH_CHECK(sub_chain(ctx, P));
    URH_LAUNCH(ctx, k_sub_text<1>, (unsigned)P.nt, SUB_THREADS, 0, P.col, n, P.ent[0], P.nt, P.next, P.cnt, d_out, capacity, (int64_t)0,
               (int64_t)0);
    URH_CHECK(sub_offset(ctx, P, P.nt, h_bytes));
    if (*h_bytes > capacity - 32) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: body of %lld bytes above its bound", (long long)*h_bytes);
    return URH_OK;
}

extern "C" int urh_sub_export_stream(urh_ctx* ctx, const void* h_iq, int dtype, int64_t n, int fd, int64_t chunk_samples, int ring,
                                     int64_t* h_bytes) {
    if (!h_iq || !h_bytes || n <= 0 || fd < 0) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export_stream: bad arguments");
    const int src_b = urh_iq_bytes(dtype);
    if (src_b == 0) URH_FAIL(ctx, URH_ERR_DTYPE, "Data type not supported");
    if (urh_div_up(n, SUB_T) >= (1ll << 31)) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: capture too long");
    URH_CHECK(urh_filter_stream_check(ctx, n, ring));
    urh_arena_reset(ctx);
    SubPlan P;
    URH_CHECK(sub_plan(ctx, P, n));
    const int64_t piece_cap = sub_piece_cap(n, chunk_samples);
    uint8_t* d_piece;
    URH_CHECK(urh_arena(ctx, (size_t)piece_cap, &d_piece));
    {   // the capture through the ring: each chunk's column I to the uint8 column
        std::vector<UrhWindow> win;
        URH_CHECK(urh_filter_windows(URH_FILTER_TILES, n, n, 0, 0, chunk_samples, nullptr, nullptr, 0, win));
        const int64_t slot = r256(stream_chunk_samples(n, chunk_samples) * src_b);
        StreamRing R;
        URH_CHECK(R.init(ctx, ring, ring * slot));
        URH_CHECK(stream_run(ctx, win, R, (const char*)h_iq, src_b, R.mem, slot, false,
                             [&](int64_t, const UrhWindow& w, int s) -> int {
                                 const int64_t cnt = w.k1 - w.k0;
                                 const unsigned grid = (unsigned)min(urh_div_up(cnt, 256), (int64_t)ctx->sm_count * 32);
                                 const void* src = R.mem + s * slot;
                                 switch (dtype) {
                                     case URH_DT_I8: URH_LAUNCH(ctx, k_sub_column<int8_t>, grid, 256, 0, (const int8_t*)src, cnt, P.col + w.k0); break;
                                     case URH_DT_U8: URH_LAUNCH(ctx, k_sub_column<uint8_t>, grid, 256, 0, (const uint8_t*)src, cnt, P.col + w.k0); break;
                                     case URH_DT_I16: URH_LAUNCH(ctx, k_sub_column<int16_t>, grid, 256, 0, (const int16_t*)src, cnt, P.col + w.k0); break;
                                     case URH_DT_U16: URH_LAUNCH(ctx, k_sub_column<uint16_t>, grid, 256, 0, (const uint16_t*)src, cnt, P.col + w.k0); break;
                                     default: URH_LAUNCH(ctx, k_sub_column<float>, grid, 256, 0, (const float*)src, cnt, P.col + w.k0); break;
                                 }
                                 return URH_OK;
                             },
                             [](int64_t, const UrhWindow&, int, cudaStream_t) { return URH_OK; }));
    }
    const size_t peak = ctx->arena_peak;
    URH_CHECK(sub_tiles(ctx, P, nullptr, dtype));
    URH_CHECK(sub_chain(ctx, P));
    // the body in pieces of whole chunks of tiles: piece p is written to fd while nothing else is queued
    URH_CHECK(urh_ensure_stage(ctx, (size_t)piece_cap));
    const int64_t tiles = sub_piece_tiles(n, chunk_samples);
    int64_t at = 0;
    for (int64_t ta = 0; ta < P.nt; ta += tiles) {
        const int64_t tb = min(P.nt, ta + tiles);
        int64_t end;
        URH_CHECK(sub_offset(ctx, P, tb, &end));
        if (end - at > piece_cap - 32) URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: piece of %lld bytes above its bound", (long long)(end - at));
        URH_LAUNCH(ctx, k_sub_text<1>, (unsigned)(tb - ta), SUB_THREADS, 0, P.col, n, P.ent[0], P.nt, P.next, P.cnt, d_piece, piece_cap, ta,
                   at);
        URH_CUDA(ctx, cudaMemcpyAsync(ctx->h_stage[0], d_piece, (size_t)(end - at), cudaMemcpyDeviceToHost, ctx->stream));
        URH_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int64_t done = 0; done < end - at;) {
            const ssize_t w = write(fd, (const char*)ctx->h_stage[0] + done, (size_t)(end - at - done));
            if (w < 0) {
                if (errno == EINTR) continue;
                URH_FAIL(ctx, URH_ERR_INVALID, "sub_export: write failed: %s", strerror(errno));
            }
            done += w;
        }
        at = end;
    }
    *h_bytes = at;
    if ((size_t)ctx->arena_peak < peak) ctx->arena_peak = peak;
    return URH_OK;
}

// Device bytes of urh_sub_export (streamed = 0: the capture, the body and the scratch) or urh_sub_export_stream (the ring, the scratch
// and one body piece), by the arena rule of the streamed entries (stream_arena_bytes)
extern "C" int urh_sub_export_footprint(int64_t n, int dtype, int streamed, int64_t chunk_samples, int ring, int64_t* h_bytes) {
    const int src_b = urh_iq_bytes(dtype);
    if (!h_bytes || n < 0 || src_b == 0 || ring < 2 || ring > URH_STREAM_MAX_RING) return URH_ERR_INVALID;
    if (n == 0) {
        *h_bytes = 0;
        return URH_OK;
    }
    SubPlan P;
    sub_levels(P, n);
    if (streamed)
        *h_bytes = ring * r256(stream_chunk_samples(n, chunk_samples) * src_b) + stream_arena_bytes(P.bytes() + sub_piece_cap(n, chunk_samples));
    else
        *h_bytes = n * src_b + r256(urh_sub_export_bound(n)) + stream_arena_bytes(P.bytes());
    return URH_OK;
}
