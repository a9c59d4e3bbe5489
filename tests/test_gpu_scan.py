"""GPU: the look-back scan (tilescan.cuh), the library's one device-wide scan, against exact host prefixes.

The primitive runs through urh_selftest_scan with the three element types of test_scan_reference_cpu (int64 sums, RunCarry
under RunCarryOp, 2x2 uint64 matrix products: 8, 16 and 32 bytes, the last the full SLOT) at every ITEMS the library uses.
A scan block covers C = 256 * ITEMS elements; the sizes sit on block edges, on 32 and 33 blocks (the look-back folds 32
predecessors per round) and past them, and `delay_chunk` holds one block back so the blocks after it fold aggregate-only
windows and take a second round.  Workspace growth (8192 blocks) and back-to-back launches without a sync are pinned too.
The second half runs every user of the scan past one scan block against the oracle or the loop-free bits model."""
import ctypes as C

import numpy as np
import pytest

from test_scan_reference_cpu import RC_DTYPE, i64_prefixes, mat_prefixes, random_mats, rc_prefixes

pytestmark = pytest.mark.gpu

ITEMS = (4, 8, 16)
OP_I64, OP_RC, OP_MAT = 0, 1, 2
GROW_BLOCKS = 8192   # a fresh context's scan workspace (context.cu urhts::prepare)


def chunk(items):
    return 256 * items


def sizes(items):
    c = chunk(items)
    return [1, 2, c - 1, c, c + 1, 32 * c, 33 * c + 1, 34 * c + 1, 100 * c + 7]


def delays(n, items):
    nb = -(-n // chunk(items))
    return [-1, 0] + ([40] if nb > 40 else [])


def make_input(op, n, items, rng):
    """host table of n elements, built so that a reordered, dropped or repeated element changes some prefix"""
    c = chunk(items)
    if op == OP_I64:
        x = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)   # both signs, totals far past 2^32
        x[rng.random(n) < 0.3] += 1 << 36                          # a drift, so partial sums differ from block to block
        return x
    if op == OP_MAT:
        return random_mats(rng, n)
    x = np.zeros(n, RC_DTYPE)
    x["len"] = rng.integers(0, 1 << 20, n)
    x["cls"] = rng.integers(0, 3, n)
    x["flags"] = rng.choice([0, 1, 1, 1, 1, 1, 2, 3], n)   # mostly whole elements: runs that cross elements; some identities
    # a class change on the first and on the last element of every block
    for b0 in range(0, n, c):
        for i in (b0, min(b0 + c, n) - 1):
            if i > 0:
                x["cls"][i] = (x["cls"][i - 1] + 1) % 3
                x["flags"][i] = 1
    if n > 34 * c:
        # one whole-span run through more than 33 blocks whose lengths sum past 2^31 (identities inside it drop out)
        lo, hi = c // 2, min(n, c // 2 + 34 * c)
        x["cls"][lo:hi] = 2
        x["flags"][lo:hi] = np.where(rng.random(hi - lo) < 0.02, 2, 1)
        x["len"][lo:hi] = rng.integers(1 << 16, 1 << 17, hi - lo)
        x["flags"][lo] = 0   # the run starts here
    return x


def reference(op, x):
    if op == OP_I64:
        e, t = i64_prefixes(x)
        return e, np.array([t], np.int64)
    if op == OP_RC:
        return rc_prefixes(x)
    e, t = mat_prefixes(x)
    return e, t.reshape(1, 4)


def words(a):
    return np.ascontiguousarray(a).view(np.uint32).reshape(-1)


class Launch:
    """one urh_selftest_scan: its device buffers (uploaded, which synchronises) and, after go(), the queued scan"""

    def __init__(self, ctx, op, items, x, delay, in_place, total=True):
        from urh_b200.device import DeviceArray, to_device

        self.ctx, self.op, self.items, self.x, self.delay, self.in_place = ctx, op, items, x, delay, in_place
        n = len(x)
        self.d_in = to_device(x, ctx)
        self.d_excl = self.d_in if in_place else DeviceArray(ctx, x.shape, x.dtype)
        self.d_elem = None if in_place else DeviceArray(ctx, x.shape, x.dtype)
        self.d_total = None
        if total:
            self.d_total = DeviceArray(ctx, (1,) + x.shape[1:], x.dtype)
            self.d_total.set(np.frombuffer(b"\xab" * self.d_total.nbytes, x.dtype).reshape(self.d_total.shape))
        self.d_held = DeviceArray(ctx, (1,), np.int32).set(np.array([-1], np.int32))

    def go(self):
        """enqueue the scan (no synchronisation)"""
        ptr = lambda d: C.c_void_p(d.ptr) if d is not None else None
        self.ctx.check(self.ctx.lib.urh_selftest_scan(self.ctx.handle, self.op, self.items, ptr(self.d_in), len(self.x), ptr(self.d_excl),
                                                      ptr(self.d_elem), ptr(self.d_total), int(self.delay),
                                                      ptr(self.d_held)))
        return self

    def check(self, ref=None):
        what = (self.op, self.items, len(self.x), self.delay, self.in_place)
        excl, total = ref or reference(self.op, self.x)
        got = self.d_excl.get()
        assert np.array_equal(words(got), words(excl)), ("excl", what, int(np.argmax(words(got) != words(excl))))
        if self.d_elem is not None:
            assert np.array_equal(words(self.d_elem.get()), words(self.x)), ("elem", what)
        if self.d_total is not None:
            assert np.array_equal(words(self.d_total.get()), words(total)), ("total", what)
        # the held block saw the next 33 blocks (or all there are) publish their aggregates before it loaded: the look-back past it
        # (a second round for the 33rd) did run
        nb = -(-len(self.x) // chunk(self.items))
        assert self.d_held.get()[0] == (1 if 0 <= self.delay < nb else -1), ("held", what)
        for d in (self.d_in, self.d_excl, self.d_elem, self.d_total, self.d_held):
            if d is not None:
                d.free()


@pytest.mark.parametrize("items", ITEMS)
@pytest.mark.parametrize("op", [OP_I64, OP_RC, OP_MAT])
def test_scan_matches_host_prefixes(ctx, op, items):
    """every size edge x {no delay, block 0 held back, block 40 held back} x {in place, separate output with d_elem}"""
    rng = np.random.default_rng(100 * op + items)
    for n in sizes(items):
        x = make_input(op, n, items, rng)
        ref = reference(op, x)
        for delay in delays(n, items):
            for in_place in (True, False):
                Launch(ctx, op, items, x, delay, in_place).go().check(ref)


def test_scan_n0_launches_nothing_and_total_may_be_null(ctx):
    from urh_b200.device import DeviceArray

    for op, dt, shape in ((OP_I64, np.int64, (4,)), (OP_RC, RC_DTYPE, (4,)), (OP_MAT, np.uint64, (4, 4))):
        d_in, d_out, d_total = DeviceArray(ctx, shape, dt), DeviceArray(ctx, shape, dt), DeviceArray(ctx, (1,) + shape[1:], dt)
        sentinel = np.frombuffer(b"\x5a" * d_total.nbytes, dt).reshape(d_total.shape)
        d_total.set(sentinel)
        for items in ITEMS:
            before = ctx.launch_count()
            ctx.check(ctx.lib.urh_selftest_scan(ctx.handle, op, items, C.c_void_p(d_in.ptr), 0, C.c_void_p(d_out.ptr), None,
                                                C.c_void_p(d_total.ptr), 0, None))
            assert ctx.launch_count() == before
        assert words(d_total.get()).tolist() == words(sentinel).tolist()
    rng = np.random.default_rng(5)
    for op in (OP_I64, OP_RC, OP_MAT):
        for items in ITEMS:
            x = make_input(op, 34 * chunk(items) + 1, items, rng)
            Launch(ctx, op, items, x, 0, False, total=False).go().check()
            Launch(ctx, op, items, x, -1, True, total=False).go().check()


def test_scan_rejects_unknown_op_and_items(ctx):
    from urh_b200.device import DeviceArray

    d = DeviceArray(ctx, (8,), np.int64)
    for op, items in ((3, 8), (-1, 8), (0, 2), (1, 32), (2, 0)):
        with pytest.raises(ValueError):
            ctx.check(ctx.lib.urh_selftest_scan(ctx.handle, op, items, C.c_void_p(d.ptr), 8, C.c_void_p(d.ptr), None, None, -1, None))


@pytest.mark.parametrize("op,items", [(OP_I64, 4), (OP_I64, 8), (OP_I64, 16), (OP_RC, 4), (OP_RC, 8), (OP_RC, 16), (OP_MAT, 4)])
def test_scan_workspace_growth(op, items):
    """a fresh context: small, 8192 blocks (fits), 8192 blocks + 1 element (grows: sync, reallocation, counter and epoch reset),
    small again with block 0 held back.  A second growth past the doubled workspace (16448 blocks) runs for int64 and RunCarry at
    ITEMS 4 only: growth is counted in blocks and prepare() does not see ITEMS or the element size, while the same step costs 67 M
    RunCarry elements at ITEMS 16 and a 16.8 M-matrix host doubling scan for the matrix op."""
    from urh_b200 import _lib

    c = chunk(items)
    rng = np.random.default_rng(7 * op + items)
    ctx = _lib.Context()
    try:
        plan = [(3 * c + 5, 0), (GROW_BLOCKS * c, -1), (GROW_BLOCKS * c + 1, 40), (34 * c + 1, 0)]
        if items == 4 and op != OP_MAT:   # the doubled workspace holds 16448 blocks
            plan += [(16449 * c - 3, -1), (100 * c + 7, 0)]
        for n, delay in plan:
            Launch(ctx, op, items, make_input(op, n, items, rng), delay, False).go().check()
    finally:
        ctx.close()


def test_scan_back_to_back_launches():
    """about 300 scans queued on one context without a sync (mixed operators, ITEMS, sizes and delays, one workspace growth
    among them); every result checked after one sync"""
    from urh_b200 import _lib

    rng = np.random.default_rng(11)
    ctx = _lib.Context()
    try:
        queued = []
        for k in range(300):
            op = int(rng.integers(0, 3))
            items = int(rng.choice(ITEMS))
            c = chunk(items)
            if k == 150:
                op, items, n, delay = OP_I64, 4, GROW_BLOCKS * 1024 + 1, 0
            else:
                n = int(rng.choice([1, 2, c - 1, c, c + 1, 33 * c + 1, 34 * c + 1, int(rng.integers(1, 50 * c))]))
                nb = -(-n // c)
                delay = int(rng.choice([-1, -1, 0, 0, 40 if nb > 40 else nb - 1]))
            queued.append(Launch(ctx, op, items, make_input(op, n, items, rng), delay, bool(rng.integers(0, 2))))
        for q in queued:   # the uploads above synchronise; the launches do not
            q.go()
        ctx.sync()
        for q in queued:
            q.check()
    finally:
        ctx.close()


# ---- every user of the scan past one scan block ------------------------------------------------------------------------------------------
TILE = 2048                     # samples per tile of the segmenter, the plateau RLE and the digitizer (dense.cuh URH_TILE)
SEG_BLOCK = 4096 * TILE         # samples per scan block of their per-tile tables (ITEMS 16)


def levels_from_edges(n, edges, dtype):
    """magnitudes: 0.9 inside [edges[2j], edges[2j + 1]), 0.05 elsewhere"""
    m = np.full(n, 0.05, dtype)
    for a, b in zip(edges[0::2], edges[1::2]):
        m[a:b] = 0.9
    return m


def seg_edges(n, rng):
    """message edges on the first and the last sample of scan blocks, plus random messages in between"""
    e = set()
    for b in range(SEG_BLOCK, n, SEG_BLOCK):
        e.update((b - 1, b))
        e.update((b - TILE * 3 + 1, b + TILE * 5 - 1))
    e.update(int(v) for v in rng.integers(1, n - 1, 64))
    e = sorted(v for v in e if 0 < v < n)
    return e[: len(e) // 2 * 2]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_segmenter_around_one_scan_block(ctx, oracle, dtype):
    from urh_b200.ainterpretation import AutoInterpretation as AI

    rng = np.random.default_rng(21)
    for n in (SEG_BLOCK - TILE - 1, SEG_BLOCK - 1, SEG_BLOCK, SEG_BLOCK + 1, SEG_BLOCK + TILE + 1, 2 * SEG_BLOCK + 1):
        mags = levels_from_edges(n, seg_edges(n, rng), dtype)
        assert AI.segment_messages_from_magnitudes(mags, 0.5) == oracle.segment_messages_from_magnitudes(mags, 0.5), n


def test_segmenter_silence_over_33_scan_blocks(ctx, oracle):
    """messages in the first scan blocks, then silence through 33 whole blocks to the end of the capture: the closing run (and the
    last segment's end) is folded across look-back rounds"""
    from urh_b200.ainterpretation import AutoInterpretation as AI

    n = 34 * SEG_BLOCK + 12345
    rng = np.random.default_rng(22)
    head = seg_edges(SEG_BLOCK + 1, rng)
    mags = levels_from_edges(n, head + [SEG_BLOCK - 7, SEG_BLOCK + 2000], np.float32)
    got = AI.segment_messages_from_magnitudes(mags, 0.5)
    assert got == oracle.segment_messages_from_magnitudes(mags, 0.5)
    # and one message that runs through 34 blocks to the end
    mags[SEG_BLOCK + 4000:] = 0.9
    assert AI.segment_messages_from_magnitudes(mags, 0.5) == oracle.segment_messages_from_magnitudes(mags, 0.5)


def test_segmenter_streamed_in_chunks_past_one_scan_block(ctx, oracle):
    """segment_messages_iq streamed with chunks longer than one scan block: each chunk's head candidates fold the carry of the
    chunks before it in front of the chunk's own prefix"""
    from urh_b200.ainterpretation import AutoInterpretation as AI

    n = 3 * SEG_BLOCK + 5 * TILE + 3
    rng = np.random.default_rng(23)
    edges = seg_edges(n, rng)
    chunk = SEG_BLOCK + 3 * TILE
    # a message across the first chunk edge and silence across the second
    edges = sorted(set(edges + [chunk - 100, chunk + 5 * TILE + 17]))
    edges = edges[: len(edges) // 2 * 2]
    mags = levels_from_edges(n, edges, np.float32)
    iq = np.zeros((n, 2), np.float32)
    phase = 2 * np.pi * rng.random(n)
    iq[:, 0] = mags * np.cos(phase)
    iq[:, 1] = mags * np.sin(phase)
    thr = 0.5
    want = oracle.segment_messages_from_magnitudes(oracle.get_magnitudes(iq), thr)
    assert AI.segment_messages_iq(iq, thr) == want
    for ch in (chunk, 2 * SEG_BLOCK + TILE):
        k = C.c_int64(-1)
        ctx.check(ctx.lib.urh_segment_messages_iq_stream(ctx.handle, iq.ctypes.data_as(C.c_void_p), 4, n, float(thr), ch, 2, C.byref(k)))
        seg = np.empty((k.value, 2), np.int64)
        ctx.check(ctx.lib.urh_fetch_segments(ctx.handle, seg.ctypes.data_as(C.c_void_p), k.value))
        assert [(int(a), int(b)) for a, b in seg] == want, ch


def test_plateau_lengths_past_one_scan_block(ctx, oracle):
    from urh_b200.cythonext import auto_interpretation as cai

    rng = np.random.default_rng(24)
    for n in (SEG_BLOCK - 1, SEG_BLOCK + 1, 2 * SEG_BLOCK + TILE + 1):
        # plateaus of random length, with level changes on the first and last sample of every scan block
        cuts = np.unique(np.concatenate([np.cumsum(rng.integers(1, 3000, n // 1000)),
                                         np.arange(SEG_BLOCK, n, SEG_BLOCK), np.arange(SEG_BLOCK, n, SEG_BLOCK) - 1]))
        cuts = cuts[(cuts > 0) & (cuts < n)]
        lv = np.repeat(rng.choice([-1.0, 1.0, 0.5, -0.25], len(cuts) + 1), np.diff(np.concatenate([[0], cuts, [n]])))
        rect = lv.astype(np.float32)
        for pct in (25, 100):
            assert np.array_equal(cai.get_plateau_lengths(rect, 0.0, pct), oracle.get_plateau_lengths(rect, 0.0, pct)), (n, pct)
    # one plateau through 33 whole scan blocks to the end
    n = 34 * SEG_BLOCK + 77
    rect = np.full(n, 1.0, np.float32)
    rect[: SEG_BLOCK // 2: 1000] = -1.0
    assert np.array_equal(cai.get_plateau_lengths(rect, 0.0, 100), oracle.get_plateau_lengths(rect, 0.0, 100))


# ---- ppseq_to_bits (four scans at ITEMS 8: 2048 rows per block) ---------------------------------------------------------------------------
PP_BLOCK = 2048


def pp_table(k, rng, sps=100, bps=1, pt=8):
    """rows of k: data rows of 0-5 symbols, short and long pauses, long pauses on the last and first row of scan blocks, a message
    running through 34 blocks without a long pause, and long pauses of 2^30 samples so the sample totals pass 2^32"""
    kinds = rng.integers(-1, 1 << bps, k)
    ns = rng.integers(0, 5 * sps + 1, k)
    long_ = rng.random(k) < 0.01
    kinds[long_] = -1
    ns[long_] = rng.integers(9, 40, int(long_.sum())) * sps
    for b in range(PP_BLOCK, k, PP_BLOCK):
        for i in (b - 1, b):
            kinds[i], ns[i] = -1, 20 * sps
    if k > 36 * PP_BLOCK:
        lo = PP_BLOCK + 5
        span = slice(lo, lo + 34 * PP_BLOCK)
        kinds[span] = np.where(rng.random(34 * PP_BLOCK) < 0.5, rng.integers(0, 1 << bps, 34 * PP_BLOCK), -1)
        ns[span] = rng.integers(0, 5 * sps + 1, 34 * PP_BLOCK)   # short pauses only: one message
    if pt:   # (with pause_threshold 0 every pause emits its zero bits)
        big = np.nonzero((kinds == -1) & (np.arange(k) >= 36 * PP_BLOCK))[0]
        ns[big[:: max(1, len(big) // 8)]] = 1 << 30
    return np.stack([kinds, ns], axis=1).astype(np.int64)


def pp_check(rows, sps, bps, pt, write_pos, ctx=None):
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import to_device
    from test_bits_model import model

    d = to_device(rows, ctx)
    bits, off, pauses, pos = sf.ppseq_to_bits(d, sps, bps, write_bit_sample_pos=write_pos, pause_threshold=pt)
    mb, moff, mp, mpos = model(rows, sps, bps, pt)
    assert np.array_equal(bits, mb) and np.array_equal(off, moff) and np.array_equal(pauses, mp), (len(rows), pt, write_pos)
    if write_pos:
        assert np.array_equal(pos, mpos), (len(rows), pt)
    d.free()


def test_ppseq_to_bits_past_scan_blocks(ctx):
    rng = np.random.default_rng(31)
    for k in (PP_BLOCK - 1, PP_BLOCK, PP_BLOCK + 1, 33 * PP_BLOCK + 1, 40 * PP_BLOCK - 1, 37 * PP_BLOCK + 11):
        for bps, pt in ((1, 8), (2, 0), (3, 1)):
            rows = pp_table(k, rng, sps=100, bps=bps, pt=pt)
            for write_pos in (True, False):
                pp_check(rows, 100, bps, pt, write_pos)
    # k = 2048 m - 1 rows: the segment-flag scan over k + 1 entries ends exactly on a block edge
    rows = pp_table(40 * PP_BLOCK - 1, rng)
    rows[-1] = (-1, 5000)   # the table ends with a long pause: an empty last segment
    pp_check(rows, 100, 1, 8, True)


def test_ppseq_to_bits_grows_the_workspace():
    """2^24 + 1 rows (8193 scan blocks) on a context that has run a small scan: its first scan grows the workspace"""
    from urh_b200 import _lib

    rng = np.random.default_rng(32)
    ctx = _lib.Context()
    try:
        pp_check(pp_table(5000, rng), 100, 1, 8, True, ctx)
        pp_check(pp_table((1 << 24) + 1, rng), 100, 1, 8, True, ctx)
        pp_check(pp_table(70001, rng), 100, 2, 8, False, ctx)
    finally:
        ctx.close()


# ---- the pulse-table finish (finish.cu) ---------------------------------------------------------------------------------------------------
def test_finish_fsk_past_34_candidate_scan_blocks(oracle):
    """an FSK capture of 34 blocks of the ITEMS-4 candidate and firing scans (1024 tiles each) plus an odd tail, with a silence over
    two whole blocks of the ITEMS-16 run-carry scan: the whole pulse table, with a given and with a detected center"""
    from conftest import synth_fsk
    from urh_b200.cythonext import signal_functions as sf

    n = 34 * 1024 * TILE + 12345
    iq = synth_fsk(n, sps=100, seed=41, gap_every=3_000_001)
    iq[SEG_BLOCK - 77: 3 * SEG_BLOCK + 5000] *= np.float32(0.001)   # run-carry blocks 1 and 2 wholly silent
    qad, rows = sf.demod_digitize(iq, 0.05, "FSK", 0.0, 5, 100)
    qad_ref = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert np.array_equal(qad.view(np.uint32), qad_ref.view(np.uint32))
    assert np.array_equal(rows, oracle.grab_pulse_lens(qad_ref, 0.0, 5, "FSK", 100))
    center, rows2 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100)
    # the one-call step takes the window variance in float64 where that may stand in for np.var's float32 pairwise sums
    # (AutoInterpretation.fused_window_stats), so its center is within 2e-6 of the reference's, the bound test_gpu_stats pins;
    # the stand-alone detect_center below is compared bit for bit.  The pulse table is exact for the center the step chose.
    assert center is not None and abs(center - oracle.detect_center(qad_ref)) <= 2e-6
    assert np.array_equal(rows2, oracle.grab_pulse_lens(qad_ref, center, 5, "FSK", 100))


def ask_capture(n_rows, rng):
    """ASK bursts: rows of 3..100 samples at amplitude 1.0 or 0.1 (short pauses and pulses under the tolerance among them)"""
    lens = rng.integers(3, 101, n_rows)
    short = rng.random(n_rows) < 0.05
    lens[short] = rng.integers(1, 5, int(short.sum()))
    amp = np.repeat(np.where(np.arange(n_rows) % 2 == 0, 1.0, 0.1), lens)
    n = len(amp)
    x = amp * np.exp(2j * np.pi * (0.01 * np.arange(n) + rng.random())) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))


def test_finish_ask_merge_past_34_scan_blocks(oracle):
    """an ASK capture whose pulse table has more than 34 x 4096 rows, so the row-merge scan (ITEMS 16) runs past 34 blocks: the
    whole table with a given and with a detected center"""
    from urh_b200.cythonext import signal_functions as sf

    iq = ask_capture(200_001, np.random.default_rng(42))
    qad_ref = oracle.afp_demod(iq, 0.05, "ASK", 2)
    rows_ref = oracle.grab_pulse_lens(qad_ref, 0.5, 5, "ASK", 50)
    assert len(rows_ref) > 34 * 4096
    qad, rows = sf.demod_digitize(iq, 0.05, "ASK", 0.5, 5, 50)
    assert np.array_equal(qad.view(np.uint32), qad_ref.view(np.uint32))
    assert np.array_equal(rows, rows_ref)
    center, rows2 = sf.demod_center_digitize(iq, 0.05, "ASK", 5, 50)
    assert center is not None and abs(center - oracle.detect_center(qad_ref)) <= 2e-6   # see the FSK case above
    assert np.array_equal(rows2, oracle.grab_pulse_lens(qad_ref, center, 5, "ASK", 50))


# ---- stand-alone detect_center (kept-count prefix over tiles, ITEMS 16: 4096 tiles per block) ---------------------------------------------
def test_detect_center_over_several_kept_count_blocks(oracle):
    """demodulated data of three scan blocks of tiles plus an odd tail; blocks 0 and 1 hold almost only samples at or below -4
    (dropped), so the kept rank window starts in block 2; bit-identical to the reference's detect_center"""
    from urh_b200.ainterpretation import AutoInterpretation as AI

    rng = np.random.default_rng(51)
    n = 3 * SEG_BLOCK + 4 * TILE + 77
    sym = np.repeat(rng.choice([-0.31, 0.27], n // 40 + 1), 40)[:n]
    x = (sym + 0.02 * rng.standard_normal(n)).astype(np.float32)
    x[:2 * SEG_BLOCK] = np.where(rng.random(2 * SEG_BLOCK) < 0.5, np.float32(-4.0), np.float32(-7.5))
    keep = rng.integers(0, 2 * SEG_BLOCK, 5000)
    x[keep] = np.float32(0.27)
    x[SEG_BLOCK - 1] = x[SEG_BLOCK] = np.float32(-0.31)   # kept samples on the edge of blocks 0 and 1
    for max_size in (None, 5000, SEG_BLOCK + 3):
        got = AI.detect_center(x, max_size)
        want = oracle.detect_center(x, max_size)
        assert (got is None) == (want is None) and (got is None or float(got) == float(want)), (max_size, got, want)


# ---- modulation_features / detect_modulation (keep-flag compaction, ITEMS 8: 2048 samples per block) ------------------------------------
MOD_BLOCK = 2048


def abs_max(x):
    """|max| of the kept samples: numpy's lexicographic complex maximum, and its magnitude rounded once from float64 (what libm's
    hypotf returns and the library reports; numpy's vectorised complex64 abs can sit 1 ulp away, which FEATURE_RATIO absorbs)"""
    m = np.max(x[np.abs(x) > 0])
    return float(np.float32(np.sqrt(np.float64(m.real) ** 2 + np.float64(m.imag) ** 2)))


def mod_message(n, zeros, rng, kind=0):
    """a complex64 message (kind 0 FSK-like, 1 ASK-like, 2 PSK-like, 3 one carrier, as test_gpu_modulation draws them) with exact
    zeros at `zeros` and a unique lexicographic maximum 3+4j right after the first zero that lies past a block edge"""
    t = np.arange(n)
    if kind == 0:
        x = np.exp(2j * np.pi * np.cumsum(np.repeat(rng.choice([-0.05, 0.05], n // 50 + 1), 50)[:n]))
    elif kind == 1:
        x = (np.repeat(rng.integers(0, 2, n // 40 + 1), 40)[:n] * 0.8 + 0.2) * np.exp(2j * np.pi * 0.01 * t)
    elif kind == 2:
        x = np.exp(1j * np.pi * np.repeat(rng.integers(0, 2, n // 30 + 1), 30)[:n]) * np.exp(2j * np.pi * 0.002 * t)
    else:
        x = np.exp(2j * np.pi * 0.03 * t)
    x = (x + 0.02 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    zeros = sorted(set(z for z in zeros if 0 <= z < n))
    x[zeros] = 0
    past = [z for z in zeros if z >= MOD_BLOCK and z + 1 < n and z + 1 not in zeros]
    if past:
        x[past[0] + 1] = 3 + 4j
    return x


def test_modulation_features_past_scan_blocks(oracle):
    from test_gpu_autointerp import FEATURE_RATIO
    from urh_b200.ainterpretation import AutoInterpretation as AI

    rng = np.random.default_rng(61)
    C_ = MOD_BLOCK
    msgs = []
    for n in (C_ - 1, C_, C_ + 1, 2 * C_ + 1, 33 * C_ + 1, 34 * C_ + 1, 40 * C_ - 1):
        for j, zeros in enumerate(([], [0], [C_ - 1, C_], [0, C_, n - 1], [C_, n - 1], [C_ - 1, C_, C_ + 2, n - 1])):
            msgs.append(mod_message(n, zeros, rng, kind=(j + len(msgs)) % 4))
    rel_dev, rel_ref = [], []
    for x in msgs:
        feat, _ = AI.modulation_features(x)
        data = x[np.abs(x) > 0]
        nz = len(data)
        assert int(feat[0]) == nz
        assert AI.detect_modulation(x) == oracle.detect_modulation(x)
        if nz == 0 or len(x) - nz > 3:
            continue
        P = 1 << int(np.log2(nz))
        assert int(feat[1]) == P and int(feat[2]) == max(P - 16, 0)
        assert feat[7] == abs_max(x)
        _, ref = oracle.modulation_features(x)
        _, truth = oracle.modulation_features(x.astype(np.complex128))
        ref, truth = np.array(ref[:4]), np.array(truth[:4])
        rel_dev.append(np.abs(feat[3:7] - truth) / np.abs(truth))
        rel_ref.append(np.abs(ref - truth) / np.abs(truth))
    assert len(rel_dev) > 30
    # FEATURE_RATIO x the complex64 reference's worst error over this set, per feature.  On these long, clean messages the
    # reference's pairwise float32 sums can land far under one float32 rounding for a feature (3e-8 for var_norm_mag while it
    # reaches 4e-7 on another), so its worst error counts as at least two float32 epsilons: a float32 result is not held closer
    # to the truth than two roundings.
    worst_ref = np.maximum(np.max(rel_ref, axis=0), 2 * np.finfo(np.float32).eps)
    assert np.all(np.array(rel_dev) <= FEATURE_RATIO * worst_ref), (np.max(rel_dev, axis=0), np.max(rel_ref, axis=0))


def test_modulation_features_grow_the_workspace(oracle):
    """a 2^24 + 1-sample message (8193 scan blocks) on a context that has run a small scan: the compaction scan grows the
    workspace inside the call"""
    from urh_b200 import _lib
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.device import to_device

    rng = np.random.default_rng(62)
    ctx = _lib.Context()
    try:
        small = mod_message(5000, [MOD_BLOCK], rng)
        feat, _ = AI.modulation_features(to_device(small, ctx))
        assert int(feat[0]) == 4999
        n = (1 << 24) + 1
        x = mod_message(n, [0, MOD_BLOCK - 1, n - 1], rng)
        feat, _ = AI.modulation_features(to_device(x, ctx))
        assert int(feat[0]) == n - 3 and int(feat[1]) == 1 << 23 and int(feat[2]) == (1 << 23) - 16
        assert feat[7] == abs_max(x)
        _, ref = oracle.modulation_features(x)
        assert np.allclose(feat[3:7], ref[:4], rtol=2e-4, atol=1e-7), (feat[3:7], ref)
    finally:
        ctx.close()
