"""GPU (one device): urh_b200.dist rank by rank, W = 1, 2, 3, 5 and 8 ranks as threads of this process (tests/one_gpu_world.py),
against the single-GPU public function on the whole capture.

Each path runs with two kinds of bounds: ``shard_bounds`` (tile-aligned) and uneven bounds with shard edges planted where shard
edges can change the answer (chunk boundaries of the noise level, run edges of the segmenter, the center's rank window, gaps and
locks of the Costas loop, message starts of estimate(), halos exactly as long as a neighbour's shard).  dist.py's plans, halo
exchanges, folds and host logic all run; only the five NCCL entry points it calls from Python are host stand-ins.

Out of scope here, because they call NCCL from inside the library: ``urh_shard_digitize`` (``demod_digitize_distributed``),
``urh_shard_demod_center_digitize(_host)`` (``demod_center_digitize_distributed``) and the center chain's rank/world mode.  They
stay with tests/test_gpu_dist.py on two or more GPUs.

The center protocol takes its bin width from the Σ/Σ² window partials where the single GPU replays numpy's float32 variance, so its
center is asserted to DESIGN §6's bar (the same None-ness, within one bin width), not word for word."""
import collections
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import autointerp_cases as aic  # noqa: E402
from one_gpu_world import OneGpuWorld  # noqa: E402

pytestmark = pytest.mark.gpu
WORLDS = (1, 2, 3, 5, 8)
CASES = collections.Counter()   # (path, W) -> cases run


@pytest.fixture(scope="module")
def contexts():
    from urh_b200 import _lib

    ctxs = [_lib.Context(0) for _ in range(max(WORLDS))]
    yield ctxs
    for c in ctxs:
        c.close()
    assert not [t.name for t in threading.enumerate() if t.name.startswith("urh-rank-")]


@pytest.fixture
def world(contexts, monkeypatch):
    from urh_b200 import _lib

    def make(W):
        w = OneGpuWorld(W, contexts[:W])
        w.install(monkeypatch, _lib.load_library())
        return w
    return make


def costas_halo():
    from urh_b200 import _lib
    return int(_lib.load_library().urh_costas_halo_samples())


def run(make, W, fn, path=None):
    """fn(rank, ctx, hx) on every rank -> [result per rank]"""
    w = make(W)
    if path:
        CASES[path, W] += 1
    return w.run(lambda r: fn(r, w.contexts[r], w.hx[r]))


def errors_of(make, W, fn):
    w = make(W)
    w.run(lambda r: fn(r, w.contexts[r], w.hx[r]), reraise=False)
    return w.errors


def even(n, W):
    from urh_b200 import dist as udist
    b = udist.shard_bounds(n, W)
    return b if all(e > s for s, e in b) else None


def planted(n, W, edges):
    """bound sets of W non-empty shards; every planted edge in (0, n) is a shard edge in one of them"""
    if W == 1:
        return [[(0, n)]]
    if n < W:
        return []
    edges = sorted(set(int(e) for e in edges if 0 < e < n))
    fill = [int(f) for f in np.linspace(0, n, 2 * W + 1)[1:-1]] + list(range(1, min(n, 4 * W)))
    out = []
    for i in range(0, max(1, len(edges)), W - 1):
        pick = set(edges[i:i + W - 1])
        for f in fill:
            if len(pick) == W - 1:
                break
            if 0 < f < n:
                pick.add(f)
        e = [0] + sorted(pick) + [n]
        out.append([(e[q], e[q + 1]) for q in range(W)])
    return out


def bound_sets(n, W, edges):
    b = even(n, W)
    return ([b] if b else []) + planted(n, W, edges)


def shard_of(ctx, x, bounds, r, halo=1, right=0):
    from urh_b200 import dist as udist
    lo, hi = bounds[r]
    sb = udist.ShardBuffer(ctx, hi - lo, x.dtype, halo=halo, right=right)
    sb.shard.set(np.ascontiguousarray(x[lo:hi]))
    return sb


def same_words(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---- noise level ------------------------------------------------------------------------------------------------------------
def noise_edges(n):
    cs, nch = aic._chunking(n)
    head = n - nch * cs
    e = [n - j * cs + d for j in (1, 2, nch // 2, nch - 1, nch) for d in (-1, 0, 1)]
    c0 = n - 6 * cs
    e += [c0 + cs // 3, c0 + (2 * cs) // 3]   # chunk 5 over three shards
    if head:
        e += [1, max(1, head // 2)]
    return e


def noise_captures():
    """(name, iq, recorded reference answer or None)"""
    want = aic.recorded("test_noise_level_iq_pinned")
    for i, (name, iq) in enumerate(aic.noise_iq_cases()):
        yield name, iq, want[i]
    for name, mag in aic.noise_cases():   # the chunk-mean edges, as float32 captures (m, 0)
        if mag.dtype == np.float32 and (len(mag) in (101, 200, 12_345) or name.startswith("edge_f32")):
            yield "mag:" + name, np.ascontiguousarray(np.stack([mag, np.zeros_like(mag)], 1)), None


@pytest.mark.parametrize("W", WORLDS)
def test_noise_level_sharded(world, W):
    from urh_b200 import dist as udist
    from urh_b200.ainterpretation import AutoInterpretation as AI

    bad, split3 = [], 0
    for name, iq, want in noise_captures():
        n = len(iq)
        one = AI.detect_noise_level_iq(iq)
        if want is not None and one != want:
            bad.append((name, "single GPU", one, want))
        cs, nch = aic._chunking(n)
        c0 = n - 6 * cs
        three = planted(n, W, [c0 + cs // 3, c0 + (2 * cs) // 3]) if W >= 3 and nch >= 6 and cs >= 3 else []
        split3 += sum(sum(1 for s, e in b if s < c0 + cs and e > c0) >= 3 for b in three)   # chunk 5 over three shards
        for bounds in bound_sets(n, W, noise_edges(n)) + three:
            def rank(r, ctx, hx):
                return udist.detect_noise_level_sharded(ctx, hx, shard_of(ctx, iq, bounds, r), bounds[r][0], n)
            got = run(world, W, rank, "noise")
            if any(g != one for g in got):
                bad.append((name, bounds, got, one))
    assert not bad, bad[:10]
    assert W < 3 or split3 > 10


def test_noise_level_tiny_captures(world):
    from urh_b200 import dist as udist
    iq = np.ones((3, 2), np.float32)
    for W in (1, 2, 3):
        bounds = planted(3, W, [1, 2])[0]
        got = run(world, W, lambda r, ctx, hx: udist.detect_noise_level_sharded(ctx, hx, shard_of(ctx, iq, bounds, r), bounds[r][0], 3),
                  "noise")
        assert got == [0] * W


# ---- segmentation -----------------------------------------------------------------------------------------------------------
def segment_edges(a, thr):
    c = a > thr
    ch = (np.nonzero(np.diff(c))[0] + 1).tolist()
    e = []
    for p in ch[:3] + ch[-2:]:
        e += [p, p - 1]           # a run's first sample, the previous run's last sample
    if ch:
        e += [ch[len(ch) // 2] + 1]   # with the edge at the change: a 1-sample shard
    eq = np.nonzero(a == thr)[0]
    if len(eq):
        e.append(int(eq[0]))
    bounds = np.concatenate([[0], ch, [len(a)]])
    k = int(np.argmax(np.diff(bounds)))
    s, t = int(bounds[k]), int(bounds[k + 1])
    if t - s > 4:
        e += [s + 1, s + 2, s + 3]   # whole-run shards in a row
    return e


@pytest.mark.parametrize("W", WORLDS)
def test_segments_sharded(world, W):
    from oracle.cassette import fingerprint
    from urh_b200 import dist as udist
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.device import to_device

    want = aic.recorded("test_segments_pinned")
    bad = []
    for i, (name, a, thr) in enumerate(aic.segment_cases()):
        one = AI.segment_messages_from_magnitudes(a, thr)
        if fingerprint(one) != want[i]:
            bad.append((name, "single GPU differs from the reference"))
        n = len(a)
        for bounds in bound_sets(n, W, segment_edges(a, thr)):
            def rank(r, ctx, hx):
                lo, hi = bounds[r]
                return udist.segment_messages_sharded(ctx, hx, to_device(np.ascontiguousarray(a[lo:hi]), ctx), lo, n, thr)
            got = run(world, W, rank, "segments")
            if any(g != one for g in got):
                bad.append((name, bounds, len(got[0]), len(one)))
    assert not bad, bad[:10]


# ---- center -----------------------------------------------------------------------------------------------------------------
def center_of_qad_shards(ctx, hx, d_qad, max_size):
    """detect_center_distributed's exchange (center_protocol) on a shard of a given qad array; the tile table from urh_center_stats"""
    import ctypes as C
    from urh_b200 import dist as udist
    lib = ctx.lib
    n = len(d_qad)
    st = np.zeros(7)
    ctx.check(lib.urh_center_stats(ctx.handle, C.c_void_p(d_qad.ptr), n, -1, st.ctypes.data_as(C.c_void_p)))

    def window_stats(lr0, lr1):
        w = np.zeros(5)
        ctx.check(lib.urh_center_window_stats(ctx.handle, C.c_void_p(d_qad.ptr), n, lr0, lr1, w.ctypes.data_as(C.c_void_p)))
        return w

    def histogram(lr0, lr1, edges):
        y = np.zeros(len(edges) - 1, dtype=np.int64)
        ctx.check(lib.urh_center_histogram_tiles(ctx.handle, C.c_void_p(d_qad.ptr), n, lr0, lr1, C.c_double(edges[0]),
                                                 C.c_double(edges[1] - edges[0]), len(y), y.ctypes.data_as(C.c_void_p)))
        return y

    def allreduce(y):
        y = np.ascontiguousarray(y, dtype=np.int64)
        ctx.check(lib.urh_nccl_allreduce_host_i64(ctx.handle, y.ctypes.data_as(C.c_void_p), len(y), 0))
        return y

    return udist.center_protocol(hx.rank, hx.world, int(st[0]), window_stats, histogram,
                                 lambda v: udist.nccl_allgather_wide(ctx, hx.world, v), allreduce, max_size)


def center_edges(x, max_size):
    """the rank window's first and last kept sample on an edge and one sample either side, a max_size cut, a shard with nothing kept"""
    kept = np.nonzero(x > -4)[0]
    k = len(kept)
    e = [2048, 4096]
    if k:
        r0, r1 = int(0.05 * k), int(0.95 * k)
        if max_size is not None and r1 - r0 > max_size:
            r1 = r0 + max_size
        for r in (r0, r1):
            if r < k:
                p = int(kept[r])
                e += [p, p + 1, p - 1]
        e.append(int(kept[k // 2]))
        gaps = np.nonzero(np.diff(kept) > 2)[0]
        if len(gaps):
            e += [int(kept[gaps[0]]) + 1, int(kept[gaps[0] + 1])]   # a shard of dropped samples only
    else:
        e.append(len(x) // 2)
    return e


def center_within_bar(got, one, step):
    """DESIGN §6: the same None-ness; a center within one bin width of the single GPU's (its bin width comes from Σ/Σ²)"""
    if got is None or one is None:
        return got is None and one is None
    return abs(got - one) <= step + 1e-9 * max(1.0, abs(one))


def single_gpu_step(x, max_size):
    import ctypes as C
    from urh_b200 import _lib
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.device import to_device
    ctx = _lib.default_context()
    d = to_device(np.ascontiguousarray(x, np.float32), ctx)
    st = np.zeros(7)
    ctx.check(ctx.lib.urh_center_stats(ctx.handle, C.c_void_p(d.ptr), len(x), -1 if max_size is None else int(max_size),
                                       st.ctypes.data_as(C.c_void_p)))
    edges = AI.center_bin_edges(st)
    return 0.0 if edges is None else float(edges[1] - edges[0])


@pytest.mark.parametrize("W", WORLDS)
def test_center_sharded_qad(world, W):
    import center_edge_cases
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.device import to_device

    bad, moved = [], 0
    cases = list(center_edge_cases.cases()) + [("all_silent", np.full(3 * 2048 + 5, np.float32(-4.0)), None)]
    for name, x, max_size in cases:
        one = AI.detect_center(x, max_size)
        step = single_gpu_step(x, max_size)
        for bounds in bound_sets(len(x), W, center_edges(x, max_size)):
            def rank(r, ctx, hx):
                lo, hi = bounds[r]
                return center_of_qad_shards(ctx, hx, to_device(np.ascontiguousarray(x[lo:hi]), ctx), max_size)
            got = run(world, W, rank, "center")
            if any(g != got[0] for g in got) or not center_within_bar(got[0], one, step):
                bad.append((name, bounds, got[0], one, step))
            moved += got[0] != one
    print("center: %d of the sharded centers differ from the single GPU's within the bar" % moved)
    assert not bad, bad[:20]


@pytest.mark.parametrize("W", WORLDS)
def test_detect_center_distributed(world, W):
    """afp_demod with its 1-sample halo + the capture-wide center, against AI.detect_center of the single-GPU qad"""
    from conftest import synth_fsk
    from urh_b200 import dist as udist
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import DeviceArray

    bad = []
    n = 120_011
    fsk = synth_fsk(n, sps=50, seed=3, gap_every=n // 5)
    env = np.repeat(np.random.default_rng(4).integers(0, 2, n // 40 + 1), 40)[:n] * 0.8 + 0.2
    ask = (fsk * env[:, None]).astype(np.float32)
    silent = (0.001 * np.random.default_rng(5).standard_normal((20_000, 2))).astype(np.float32)
    for name, iq, mod, noise, ms in [("fsk", fsk, "FSK", 0.05, None), ("ask", ask, "ASK", 0.05, None), ("fsk_max_size", fsk, "FSK", 0.05, 7000),
                                     ("int16_fsk", (fsk * 20000).astype(np.int16), "FSK", 1000.0, None), ("silent", silent, "ASK", 0.5, None)]:
        qad = sf.afp_demod(iq, noise, mod, 2)
        one = AI.detect_center(qad, ms)
        step = single_gpu_step(qad, ms)
        for bounds in bound_sets(len(iq), W, [n // 5, n // 5 + 4096, n // 20, len(iq) - 2048]):
            def rank(r, ctx, hx):
                sb = shard_of(ctx, iq, bounds, r)
                udist.exchange_halo(ctx, hx, sb)
                d_qad = DeviceArray(ctx, (sb.n,), np.float32)
                return udist.detect_center_distributed(ctx, r, hx.world, sb, noise, mod, d_qad, ms)
            got = run(world, W, rank, "detect_center_distributed")
            if any(g != got[0] for g in got) or not center_within_bar(got[0], one, step):
                bad.append((name, bounds, got[0], one, step))
    assert not bad, bad[:20]


# ---- PSK --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", WORLDS)
def test_psk_sharded(world, W):
    from test_gpu_costas import synth_psk
    from urh_b200 import dist as udist
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import DeviceArray

    halo = costas_halo()
    n = 150_000
    bad = []
    for order in (2, 4):
        iq = synth_psk(n, order, seed=60 + order, gap_period=50_000, gap_len=15_000)
        ref = sf.afp_demod(iq, 0.2, "PSK", order)
        # in a gap, mid-burst, on a burst's first sample (where the loop locks), shards just above the halo
        edges = [40_000, 45_000, 50_000, 50_001, 20_017, 50_000 + halo + 1, 50_000 + 2 * halo + 3, 100_000 + halo]
        for bounds in bound_sets(n, W, edges):
            if any(e - s < halo for s, e in bounds[:-1]):
                continue   # test_shard_shorter_than_the_costas_halo_raises_on_every_rank

            def rank(r, ctx, hx):
                sb = shard_of(ctx, iq, bounds, r, halo=halo)
                udist.exchange_halo(ctx, hx, sb)
                d_out = DeviceArray(ctx, (sb.n,), np.float32)
                udist.afp_demod_psk_sharded(ctx, r, hx.world, sb, 0.2, order, 0.1, d_out)
                return d_out.get()
            got = np.concatenate(run(world, W, rank, "psk"))
            diff = np.nonzero(got[1:].view(np.uint32) != ref[1:].view(np.uint32))[0] + 1
            if len(diff):
                bad.append((order, bounds, len(diff), diff[:3].tolist()))
    assert not bad, bad[:10]


@pytest.mark.parametrize("W", (2, 3))
def test_psk_buffer_halo_shorter_than_the_warm_up_raises_on_every_rank(world, W):
    """every ShardBuffer holds a 1-sample halo: rank 0 raises with the others, before the hypothesis all-gather"""
    from urh_b200 import dist as udist
    from urh_b200.device import DeviceArray

    n = 30_000
    iq = (np.random.default_rng(2).standard_normal((n, 2))).astype(np.float32)
    bounds = planted(n, W, [])[0]
    errs = errors_of(world, W, lambda r, ctx, hx: udist.afp_demod_psk_sharded(ctx, r, hx.world, shard_of(ctx, iq, bounds, r, halo=1), 0.2, 2,
                                                                              0.1, DeviceArray(ctx, (bounds[r][1] - bounds[r][0],), np.float32)))
    assert all(isinstance(e, ValueError) and "Costas warm-up" in str(e) for e in errs), errs


@pytest.mark.parametrize("W", (2, 3, 5))
@pytest.mark.parametrize("short", ("first", "middle"))
def test_shard_shorter_than_the_costas_halo_raises_on_every_rank(world, W, short):
    from urh_b200 import dist as udist
    from urh_b200.device import DeviceArray

    halo = costas_halo()
    n = 20_000
    iq = (np.random.default_rng(1).standard_normal((n, 2))).astype(np.float32)
    q = 0 if short == "first" else max(0, W // 2 - 1) + (W > 3)   # a shard that supplies a halo (not the last)
    lens = [(n - (halo - 1)) // (W - 1)] * W
    lens[q] = halo - 1
    lens[-1] = n - sum(lens[:-1])
    cuts = np.concatenate([[0], np.cumsum(lens)]).astype(int)
    bounds = [(int(cuts[r]), int(cuts[r + 1])) for r in range(W)]

    def rank(r, ctx, hx):
        sb = shard_of(ctx, iq, bounds, r, halo=halo)
        udist.exchange_halo(ctx, hx, sb)
        udist.afp_demod_psk_sharded(ctx, r, hx.world, sb, 0.2, 2, 0.1, DeviceArray(ctx, (sb.n,), np.float32))

    errs = errors_of(world, W, rank)
    CASES["psk", W] += 1
    assert all(isinstance(e, ValueError) for e in errs), errs
    assert len(set(str(e) for e in errs)) == 1


# ---- estimate() -------------------------------------------------------------------------------------------------------------
def estimate_captures():
    from conftest import synth_fsk
    from test_gpu_costas import synth_psk

    n = 240_000
    rng = np.random.default_rng(77)
    fsk = synth_fsk(n, sps=100, seed=91, gap_every=20_000)
    fsk[-8_000:] *= 0.001
    env = np.repeat(rng.integers(0, 2, n // 100 + 1), 100)[:n]
    ook = (synth_fsk(n, sps=100, seed=92, gap_every=30_000) * np.where(env > 0, 1.0, 0.0)[:, None]).astype(np.float32)
    ask = (synth_fsk(n, sps=100, seed=93, gap_every=30_000) * (env * 0.7 + 0.3)[:, None]).astype(np.float32)
    psk = synth_psk(n, 2, seed=94, gap_period=60_000, gap_len=18_000)
    for name, iq in (("FSK", fsk), ("OOK", ook), ("ASK", ask), ("PSK", psk)):
        yield name, np.ascontiguousarray(iq, np.float32)


@pytest.mark.parametrize("W", WORLDS)
def test_estimate_sharded(world, W):
    from urh_b200 import dist as udist
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.signalprocessing.IQArray import IQArray

    halo = costas_halo()
    bad, spans3 = [], 0
    combos = None
    for kind, iq in estimate_captures():
        n = len(iq)
        ones = {}
        noise_one = AI.detect_noise_level_iq(iq)
        msgs = AI.segment_messages_iq(iq, noise_one)
        longest = max(msgs, key=lambda m: m[1] - m[0]) if msgs else (n // 3, n // 2)
        a, b = longest
        # a message starting on an edge, one straddling an edge, the longest cut into W - 1 pieces (fetch_range over 3+ ranks),
        # and the last message owned by the last rank
        edges = [m[0] for m in msgs[1:3]] + [(m[0] + m[1]) // 2 for m in msgs[3:5]] + ([msgs[-1][0] - 1] if msgs else [])
        cut = planted(n, W, [a + (b - a) * k // (W - 1) for k in range(1, W - 1)] + [b - 1]) if W >= 3 else []
        spans3 += sum(sum(1 for s, e in q if s < b and e > a) >= 3 for q in cut)
        combos = [(None, None), (None, kind), (noise_one, None), (noise_one, kind)]
        runs = [(bounds, combos[i % 4]) for i, bounds in enumerate(bound_sets(n, W, edges) + cut)]
        if W == 1:
            runs = [(runs[0][0], c) for c in combos]
        for bounds, (noise, modulation) in runs:
            if any(e - s < halo for s, e in bounds[:-1]):
                continue
            if (noise, modulation) not in ones:
                ones[noise, modulation] = AI.estimate(IQArray(iq), noise=noise, modulation=modulation)
            one = ones[noise, modulation]

            def rank(r, ctx, hx):
                sb = shard_of(ctx, iq, bounds, r, halo=halo)
                udist.exchange_halo(ctx, hx, sb)
                return udist.estimate_sharded(ctx, hx, sb, bounds, n, noise=noise, modulation=modulation)
            got = run(world, W, rank, "estimate")
            if any(g != one for g in got):
                bad.append((kind, noise, modulation, bounds, got[0], one))
    assert not bad, bad[:10]
    assert W < 3 or spans3 >= 3   # fetch_range collected the longest message from three or more ranks


# ---- halos and fetch_range --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", (2, 3, 5, 8))
def test_halo_exchanges_and_fetch_range(world, W):
    from urh_b200 import dist as udist

    n = 3001
    x = np.random.default_rng(W).integers(-30000, 30000, (n, 2)).astype(np.int16)
    base = planted(n, W, [])[0]
    lens = [e - s for s, e in base]
    h = min(lens[:-1])   # the halo equals the shortest supplying shard: a whole neighbour's shard
    # g0 / g1 on shard edges, one sample past them, the whole capture, a whole shard, one sample; owners first, middle and last
    specs = [(base[0][1], base[-1][0] + 1, W - 1), (0, n, 0), (base[1][0] - 1, min(n, base[1][1] + 1), 1),
             (base[W // 2][0], base[W // 2][1], W // 2), (5, 6, W - 1)]

    def rank(r, ctx, hx):
        sb = shard_of(ctx, x, base, r, halo=h, right=h)
        udist.exchange_halo(ctx, hx, sb)
        left = sb.halo.get() if r else None
        halos = [(h if q else 0, h if q < W - 1 else 0) for q in range(W)]
        sb2 = shard_of(ctx, x, base, r, halo=h, right=h)
        udist.exchange_halos(ctx, hx, sb2, halos)
        ctx.sync()
        both = sb2.window(h if r else 0, h if r < W - 1 else 0).get()
        fetched = []
        for g0, g1, owner in specs:
            out = udist.fetch_range(ctx, r, base, sb.shard, g0, g1, owner)
            fetched.append(None if out is None else out.get())
        return left, both, fetched

    got = run(world, W, rank, "halos")
    for r, (left, both, fetched) in enumerate(got):
        lo, hi = base[r]
        if r:
            assert same_words(left, x[lo - h: lo]), r
        assert same_words(both, x[lo - (h if r else 0): hi + (h if r < W - 1 else 0)]), r
    for k, (g0, g1, owner) in enumerate(specs):
        for r in range(W):
            f = got[r][2][k]
            assert (f is None) == (r != owner)
            if r == owner:
                assert same_words(f, x[g0:g1]), (k, g0, g1, owner)

    # one sample too long: every rank raises before the collective
    def too_long(r, ctx, hx):
        udist.exchange_halo(ctx, hx, shard_of(ctx, x, base, r, halo=h + 1))
    errs = errors_of(world, W, too_long)
    assert all(isinstance(e, ValueError) for e in errs), errs


# ---- filters and spectrogram ------------------------------------------------------------------------------------------------
def filter_capture(n, seed, dtype=np.float32):
    rng = np.random.default_rng(seed)
    if dtype != np.float32:
        info = np.iinfo(dtype)
        return rng.integers(info.min, info.max + 1, (n, 2)).astype(dtype)
    t = np.arange(n)
    x = np.exp(2j * np.pi * 0.05 * t) * (1 + 0.5 * (rng.random(n) > 0.5)) + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    x += 0.3 - 0.2j
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))


def gathered_shards(outs):
    return np.concatenate([o for o in outs])


@pytest.mark.parametrize("W", WORLDS)
def test_filters_sharded(world, W):
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Filter import Filter, FilterType

    bad = []
    n = 60_001
    x = filter_capture(n, 1)
    xc = x.view(np.complex64).reshape(-1)
    # band-pass: 8 ln sqrt(60001) = 44, so 101 taps take the FFT branch and 41 and 31 taps the direct one
    for f_low, f_high, m in [(0.03, 0.07, 101), (0.03, 0.07, 41), (0.07, 0.03, 31)]:
        bw = Filter.get_bandwidth_from_filter_length(m)
        taps = len(Filter.bandpass_taps(f_low, f_high, bw))
        ref = Filter.apply_bandpass_filter(xc, f_low, f_high, bw).view(np.float32).reshape(-1, 2)
        half = (taps - 1) // 2
        edges = [taps - 1 - half, 2 * (taps - 1 - half), n - half, 777]   # shards exactly as long as a halo
        for bounds in bound_sets(n, W, edges):
            try:
                udist.bandpass_plan(n, taps, bounds)
            except ValueError:
                continue
            # the default output halo (the Costas warm-up) where every shard can supply it
            out_halo = 0 if any(e - s < costas_halo() for s, e in bounds[:-1]) else None

            def rank(r, ctx, hx):
                out = udist.apply_bandpass_filter_sharded(ctx, hx, shard_of(ctx, x, bounds, r), bounds, f_low, f_high, bw, out_halo)
                return out.shard.get(), (out.halo.get() if r else None)
            got = run(world, W, rank, "bandpass")
            if not same_words(gathered_shards([g for g, _ in got]), ref):
                bad.append(("band-pass", taps, bounds))
            for r in range(1, W):
                g0 = bounds[r][0]
                if out_halo is None and not same_words(got[r][1], ref[g0 - len(got[r][1]): g0]):
                    bad.append(("band-pass output halo", taps, bounds, r))
    # FIR (Filter.work) with 1, 10 and 101 taps, shards exactly m - 1 long
    for m in (1, 10, 101):
        taps = list((np.random.default_rng(m).standard_normal(m) / m).astype(np.complex64))
        ref = Filter(taps).work(x).view(np.float32).reshape(-1, 2)
        for bounds in bound_sets(n, W, [m - 1, 2 * (m - 1), 3 * (m - 1) + 1, 5000]):
            try:
                udist.fir_plan(n, m, bounds)
            except ValueError:
                continue

            def rank(r, ctx, hx):
                return udist.filter_work_sharded(ctx, hx, shard_of(ctx, x, bounds, r), bounds, Filter(taps, FilterType.custom), out_halo=0).shard.get()
            got = run(world, W, rank, "fir")
            if not same_words(gathered_shards(got), ref):
                bad.append(("fir", m, bounds))
    # DC correction: the float32 chain (bit for bit), float32 above 2^22 rows (x - float32(float64 mean)), int8 / uint16 (bit for bit)
    for nd, dtype in [(50_001, np.float32), (Filter.EXACT_DC_MAX + 3, np.float32), (40_003, np.int8), (39_999, np.uint16)]:
        xd = filter_capture(nd, nd, dtype)
        if dtype == np.float32 and nd > Filter.EXACT_DC_MAX:
            ref = xd - np.mean(xd.astype(np.float64), axis=0).astype(np.float32)
        else:
            ref = Filter.dc_correction(xd)
        for bounds in bound_sets(nd, W, [1, 2, nd // 3, nd - 1])[:3]:
            def rank(r, ctx, hx):
                return udist.filter_work_sharded(ctx, hx, shard_of(ctx, xd, bounds, r), bounds, Filter([0.1], FilterType.dc_correction),
                                                 out_halo=0).shard.get()
            got = run(world, W, rank, "dc")
            if not same_words(gathered_shards(got), ref):
                bad.append(("dc", nd, np.dtype(dtype).name, bounds))
    assert not bad, bad[:10]


@pytest.mark.parametrize("W", WORLDS)
def test_spectrogram_sharded(world, W):
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    bad = []
    n = 70_001
    x = filter_capture(n, 2)
    xc = x.view(np.complex64).reshape(-1)
    for Wn, overlap in [(1024, 0.5), (256, 0.75), (1000, 0.5)]:
        hop = Wn - int(overlap * Wn)
        ref = Spectrogram(xc, window_size=Wn, overlap_factor=overlap).calculate_spectrogram()
        # edges off the hop grid, on it, and a shard as long as the last frame's reach
        for bounds in bound_sets(n, W, [hop * 7 + 1, hop * 9, hop * 9 + Wn - hop, 3 * hop + 5]):
            try:
                udist.frame_plan(n, Wn, hop, bounds)
            except ValueError:
                continue

            def rank(r, ctx, hx):
                f0, db = udist.spectrogram_db_sharded(ctx, hx, shard_of(ctx, x, bounds, r), bounds, Wn, overlap)
                return f0, db.get()
            got = run(world, W, rank, "db")
            if not same_words(np.concatenate([d for _, d in got]), ref) or [f for f, _ in got] != sorted(f for f, _ in got):
                bad.append(("db", Wn, overlap, bounds))
    cmap = np.random.default_rng(4).integers(0, 256, (256, 4)).astype(np.uint8)
    nbig = 1_200_003
    xb = filter_capture(nbig, 5)
    for Wn, overlap, transpose in [(1024, 0.5, False), (256, 0.75, True)]:
        spec = Spectrogram(xb.view(np.complex64).reshape(-1), window_size=Wn, overlap_factor=overlap)
        segs = spec.segment_bounds()
        if transpose:
            ref = [spec.create_spectrogram_image(s, e, transpose=True, colormap=cmap) for s, e, _ in segs]
        else:
            ref = list(spec.create_image_segments(colormap=cmap))
        edges = [segs[0][1] + 1, segs[min(1, len(segs) - 1)][0], nbig // 2 + 3]
        for bounds in bound_sets(nbig, W, edges)[:2]:
            try:
                udist.segment_plan(nbig, Wn, spec.hop_size, bounds)
            except ValueError:
                continue

            def rank(r, ctx, hx):
                mine = udist.spectrogram_image_segments_sharded(ctx, hx, shard_of(ctx, xb, bounds, r), bounds, Wn, overlap, colormap=cmap,
                                                                transpose=transpose)
                return [(i, img.get()) for i, img in mine]
            got = sorted((i, img) for part in run(world, W, rank, "images") for i, img in part)
            if [i for i, _ in got] != list(range(len(ref))) or not all(same_words(a, b) for (_, a), b in zip(got, ref)):
                bad.append(("images", Wn, overlap, transpose, bounds))
    assert not bad, bad[:10]


@pytest.mark.parametrize("W", (2, 3, 5))
def test_filter_halo_one_sample_too_long_raises_on_every_rank(world, W):
    """a shard one sample shorter than the band-pass halo its neighbour needs: every rank raises ValueError, none is left waiting"""
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Filter import Filter

    n = 20_001
    x = filter_capture(n, 3)
    bw = Filter.get_bandwidth_from_filter_length(31)
    taps = len(Filter.bandpass_taps(0.03, 0.07, bw))
    need = taps - 1 - (taps - 1) // 2
    cuts = [0, need - 1] + [int(v) for v in np.linspace(need - 1, n, W)[1:]]
    bounds = [(cuts[q], cuts[q + 1]) for q in range(W)]
    errs = errors_of(world, W, lambda r, ctx, hx: udist.apply_bandpass_filter_sharded(ctx, hx, shard_of(ctx, x, bounds, r), bounds, 0.03,
                                                                                      0.07, bw))
    CASES["bandpass", W] += 1
    assert all(isinstance(e, ValueError) for e in errs), errs
    assert len(set(str(e) for e in errs)) == 1


def test_zz_cases_per_path_and_world(capsys):
    """every path ran at every world size; the table is printed"""
    if not CASES:
        pytest.skip("counts the cases of the tests above; run with them")
    paths = sorted(set(p for p, _ in CASES))
    with capsys.disabled():
        print("\ncases per path and world size (W = %s)" % ", ".join(map(str, WORLDS)))
        for p in paths:
            print("  %-26s %s" % (p, "  ".join("%5d" % CASES[p, W] for W in WORLDS)))
    for p in ("noise", "segments", "center", "detect_center_distributed", "psk", "estimate", "bandpass", "fir", "dc", "db", "images"):
        for W in WORLDS:
            assert CASES[p, W] > 0, (p, W)
