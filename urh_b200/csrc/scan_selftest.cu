// Test entry point of the look-back scan (tilescan.cuh): the library's one device-wide scan, run over a caller's table with a chosen
// element type, operator and ITEMS, so the tests can pin it against exact host prefixes at every block and look-back-round edge.
#include "common.cuh"
#include "sparse.cuh"
#include "tilescan.cuh"

// 2x2 matrix of uint64, row-major: the full SLOT, and an associative operator that is not commutative
struct __align__(16) Mat2 {
    uint64_t a[4];
};
struct Mat2Mul {
    __device__ __forceinline__ Mat2 operator()(const Mat2& x, const Mat2& y) const {   // x * y mod 2^64
        Mat2 r;
        r.a[0] = x.a[0] * y.a[0] + x.a[1] * y.a[2];
        r.a[1] = x.a[0] * y.a[1] + x.a[1] * y.a[3];
        r.a[2] = x.a[2] * y.a[0] + x.a[3] * y.a[2];
        r.a[3] = x.a[2] * y.a[1] + x.a[3] * y.a[3];
        return r;
    }
};
static_assert(sizeof(Mat2) == urhts::SLOT, "the matrix element fills the scan's SLOT");

// in[i] -> excl[i] (and elem[i]); excl may be in.  Every thread of chunk `delay_chunk` spins once, on its first element, so the
// blocks after that chunk reach their look-back while it is still running.  Its thread 0 first waits (bounded) until the next 33
// blocks have published their aggregates and reports in *held whether they all had: then the 33rd of them found 32 aggregate-only
// predecessors and went on to a second look-back round, which has to wait for this block.
template <typename T>
struct SelftestIO {
    const T* in;
    T* excl;
    T* elem;
    int64_t delay_lo, delay_hi;   // element range of the delayed chunk (empty: no delay)
    int items;
    int64_t delay_chunk, nblocks;
    const uint32_t* status;
    uint32_t epoch;
    int* held;
    __device__ __forceinline__ T load(int64_t i) const {
        if (i >= delay_lo && i < delay_hi && (i - delay_lo) % items == 0) {
            if (i == delay_lo) {
                const int64_t last = min(delay_chunk + 33, nblocks - 1);
                bool all = false;
                const long long w0 = clock64();
                while (!all && clock64() - w0 < 4000000) {   // about 2 ms at most
                    all = true;
                    for (int64_t b = delay_chunk + 1; b <= last; b++) all = all && urhts::ld_status(status + b) == ((epoch << 2) | 1u);
                }
                if (held) *held = all ? 1 : 0;
            }
            const long long t0 = clock64();
            while (clock64() - t0 < 100000) {}   // about 50 us at the H100's clock: bounded
        }
        return in[i];
    }
    __device__ __forceinline__ void post(int64_t i, const T& e, const T& v) const {
        excl[i] = e;
        if (elem) elem[i] = v;
    }
};

// urhts::scan with the workspace's status words and epoch handed to the load hook
template <typename T, typename Op, int ITEMS>
static int selftest_scan(urh_ctx* ctx, T identity, const void* d_in, int64_t n, void* d_excl, void* d_elem, void* d_total,
                         int64_t delay_chunk, int* d_held) {
    constexpr int64_t CHUNK = (int64_t)urhts::BLOCK * ITEMS;
    if (n <= 0) return URH_OK;
    const int64_t nb = urh_div_up(n, CHUNK);
    urhts::Ws ws;
    URH_CHECK(urhts::prepare(ctx, nb, &ws));
    SelftestIO<T> f;
    f.in = (const T*)d_in;
    f.excl = (T*)d_excl;
    f.elem = (T*)d_elem;
    f.delay_lo = delay_chunk >= 0 ? delay_chunk * CHUNK : 0;
    f.delay_hi = delay_chunk >= 0 ? (delay_chunk + 1) * CHUNK : 0;
    f.items = ITEMS;
    f.delay_chunk = delay_chunk;
    f.nblocks = nb;
    f.status = ws.status;
    f.epoch = ws.epoch;
    f.held = d_held;
    URH_LAUNCH(ctx, (urhts::k_scan<T, Op, SelftestIO<T>, ITEMS>), (unsigned)nb, urhts::BLOCK, 0, n, identity, Op(), f, ws, (T*)d_total);
    return URH_OK;
}

template <typename T, typename Op>
static int selftest_items(urh_ctx* ctx, int items, T identity, const void* d_in, int64_t n, void* d_excl, void* d_elem, void* d_total,
                          int64_t delay_chunk, int* d_held) {
    switch (items) {
        case 4: return selftest_scan<T, Op, 4>(ctx, identity, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
        case 8: return selftest_scan<T, Op, 8>(ctx, identity, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
        case 16: return selftest_scan<T, Op, 16>(ctx, identity, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
    }
    URH_FAIL(ctx, URH_ERR_INVALID, "items must be 4, 8 or 16 (got %d)", items);
}

// op 0: int64 sums; 1: RunCarry / RunCarryOp (sparse.cuh); 2: Mat2 products.  Enqueues one scan and does not synchronise.
extern "C" int urh_selftest_scan(urh_ctx* ctx, int op, int items, const void* d_in, int64_t n, void* d_excl, void* d_elem,
                                 void* d_total, int64_t delay_chunk, int* d_held) {
    if (!d_in || !d_excl) URH_FAIL(ctx, URH_ERR_INVALID, "d_in and d_excl are required");
    switch (op) {
        case 0: return selftest_items<int64_t, urhts::AddI64>(ctx, items, (int64_t)0, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
        case 1: {
            RunCarry ident;
            ident.len = 0;
            ident.cls = 0;
            ident.flags = 2 | 1;
            return selftest_items<RunCarry, RunCarryOp>(ctx, items, ident, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
        }
        case 2: {
            Mat2 ident;
            ident.a[0] = 1; ident.a[1] = 0; ident.a[2] = 0; ident.a[3] = 1;
            return selftest_items<Mat2, Mat2Mul>(ctx, items, ident, d_in, n, d_excl, d_elem, d_total, delay_chunk, d_held);
        }
    }
    URH_FAIL(ctx, URH_ERR_INVALID, "op must be 0 (int64 sum), 1 (run carry) or 2 (2x2 matrix product), got %d", op);
}
