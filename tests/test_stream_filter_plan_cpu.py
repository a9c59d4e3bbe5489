"""CPU: the plan of the windowed ring (urh_stream_windows, urh_stream_window_schedule, urh_stream_filter_footprint and the shims' path
choice) for the streamed band-pass, FIR and DC filters and the spectrogram, without a device.

Each chunk owns the outputs [k0, k1) and uploads the input window [a, b).  Checked here: the chunks cover every output once, each window
is exactly the samples its outputs read, the windows equal the sharded plans of urh_b200/dist.py where the cut is a valid shard cut, and
no slot is rewritten before its readers on a host model of the schedule's stream/event semantics (stream_window.cu): uploads run on
copy stream 0, chunk computations on the compute stream, downloads on copy stream 1, and every wait resolves to the last record of its
event issued before it, as cudaStreamWaitEvent does.  The model also takes the tile chunks of the demodulation entries
(URH_FILTER_TILES; their own plan is checked in tests/test_stream_plan_cpu.py)."""
import ctypes as C

import numpy as np
import pytest

from urh_b200 import dist as udist


@pytest.fixture(scope="module")
def L():
    from urh_b200 import _lib, build

    build.build()
    return _lib


def windows(L, entry, n, out_len, p0, p1, cs, segments=None):
    lib = L.load_library()
    count = C.c_int64(0)
    st = np.array([s for s, _ in segments] if segments else [0], dtype=np.int64)
    ln = np.array([x for _, x in segments] if segments else [0], dtype=np.int64)
    nseg = len(segments) if segments else 0
    args = (entry, n, out_len, p0, p1, cs, st.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), nseg)
    assert lib.urh_stream_windows(*args, None, 0, C.byref(count)) == 0
    w = np.zeros((max(count.value, 1), 4), np.int64)
    assert lib.urh_stream_windows(*args, w.ctypes.data_as(C.c_void_p), count.value, C.byref(count)) == 0
    return w[: count.value]


def covers_once(w, total):
    assert w[0, 0] == 0 and w[-1, 1] == total
    assert np.array_equal(w[1:, 0], w[:-1, 1])
    assert (w[:, 1] > w[:, 0]).all()


def shard_bounds_of(w):
    """the chunks' owned outputs as shard bounds (FIR, DC and the band-pass 'same' cut, where output k sits at sample k)"""
    return [(int(a), int(b)) for a, b in w[:, :2]]


CS = 1000
TILE = 2048


@pytest.mark.parametrize("n", [1, CS - 1, CS, CS + 1, 3 * CS - 1, 3 * CS, 3 * CS + 1, 7 * CS + 13])
@pytest.mark.parametrize("m", [1, 11, 101, 2501])
@pytest.mark.parametrize("where", ["same", "zero", "m-1", "past"])
def test_convolve_windows(L, n, m, where):
    offset, out_len = {"same": ((m - 1) // 2, n), "zero": (0, n + m - 1), "m-1": (m - 1, n),
                       "past": (max(0, n + m - 3), 2 * m + 5)}[where]
    w = windows(L, L.FILTER_CONVOLVE, n, out_len, m, offset, CS)
    covers_once(w, out_len)
    for k0, k1, a, b in w:
        lo, hi = max(0, k0 + offset - (m - 1)), min(n, k1 + offset)   # the samples outputs k0 .. k1 - 1 read
        assert (a, b) == ((lo, hi) if lo < hi else (b, b)), (k0, k1, a, b)
        assert b - a <= CS + m - 1
    if where == "same" and n >= m and (m < 8 * np.log(np.sqrt(n)) or m % 2):
        try:
            plan = udist.bandpass_plan(n, m, shard_bounds_of(w))
        except ValueError:
            return   # a chunk shorter than the filter's halo: not a valid shard cut
        for (k0, k1, a, b), (left, right, off) in zip(w, plan):
            assert (a, b, k0 + offset - a) == (k0 - left, k1 + right, off)


@pytest.mark.parametrize("n", [1, CS - 1, CS, CS + 1, 4 * CS - 1, 4 * CS, 4 * CS + 1])
@pytest.mark.parametrize("m", [0, 1, 2, 10, 101, 1000, 2500])
def test_fir_windows(L, n, m):
    w = windows(L, L.FILTER_FIR, n, n, m, 0, CS)
    covers_once(w, n)
    h = max(0, m - 1)
    for k0, k1, a, b in w:
        assert b == k1 and a == (k0 - h if k0 else 0)
        assert k0 == 0 or k0 >= h                       # every later chunk has its whole history in its own window
    assert (w[:-1, 1] - w[:-1, 0] == max(CS, h)).all()   # chunks are at least the history long
    hist = udist.fir_plan(n, m, shard_bounds_of(w))
    assert [int(k0 - a) for k0, _, a, _ in w] == hist


@pytest.mark.parametrize("n", [1, CS - 1, CS, CS + 1, 5 * CS + 1])
def test_dc_windows(L, n):
    w = windows(L, L.FILTER_DC, n, n, 0, 0, CS)
    covers_once(w, n)
    assert np.array_equal(w[:, :2], w[:, 2:])


def num_frames(n, W, hop):
    return max(1, (max(n, W) - W) // hop + 1)


@pytest.mark.parametrize("W,overlap", [(128, 0.0), (1000, 0.3), (1001, 0.5), (1024, 0.75), (4096, 0.5)])
@pytest.mark.parametrize("n_rel", [-1, 0, 1, 3, 17])
@pytest.mark.parametrize("cs_frames", [0, 1, 3])
def test_frame_windows(L, W, overlap, n_rel, cs_frames):
    hop = W - int(overlap * W)
    n = max(1, W + n_rel * hop + (n_rel % 5))
    frames = num_frames(n, W, hop)
    cs = cs_frames * hop + (hop // 2 if cs_frames else 1)   # 0: a chunk shorter than a hop still takes one frame
    for entry in (L.FILTER_STFT, L.FILTER_DB):
        w = windows(L, entry, n, frames, W, hop, cs)
        covers_once(w, frames)
        fpc = max(1, cs // hop)
        assert (w[:-1, 1] - w[:-1, 0] == fpc).all()
        for f0, f1, a, b in w:
            assert (a, b) == (f0 * hop, min(n, (f1 - 1) * hop + W))
    try:
        plan = udist.frame_plan(n, W, hop, [(int(a), int(b)) for a, b in zip(w[:, 2], list(w[1:, 2]) + [n])])
    except ValueError:
        return
    for (f0, f1, a, b), (pf0, pnf, right) in zip(w, plan):
        assert (pf0, pnf) == (f0, f1 - f0)


@pytest.mark.parametrize("n", [5000, 20_000, 100_003])
@pytest.mark.parametrize("W,overlap", [(128, 0.5), (256, 0.0), (1000, 0.75)])
@pytest.mark.parametrize("cs", [300, 4000, 1 << 20])
@pytest.mark.parametrize("max_lines", [3, 10, 1000])
def test_image_windows(L, n, W, overlap, cs, max_lines):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    hop = W - int(overlap * W)
    segs = Spectrogram.segment_bounds_of(n, W, hop, max_lines)
    segments = [(s, e - s) for s, e, _ in segs]
    frames = [f for _, _, f in segs]
    cum = np.concatenate([[0], np.cumsum(frames)])
    w = windows(L, L.FILTER_IMAGES, n, 0, W, hop, cs, segments)
    covers_once(w, int(cum[-1]))
    check_image_windows(w, segments, cum, W, hop, cs)
    groups = all(k1 > cum[int(np.searchsorted(cum, k0, side="right"))] or (k0, k1) in zip(cum[:-1], cum[1:]) for k0, k1, _, _ in w)
    if groups and len(w) > 1:
        bounds = [(int(a), int(b)) for a, b in zip(w[:, 2], list(w[1:, 2]) + [n])]
        try:
            _, owned, rights = udist.segment_plan(n, W, hop, bounds, max_lines)
        except ValueError:
            return
        for (k0, k1, a, b), mine, right, (g0, g1) in zip(w, owned, rights, bounds):
            assert mine == [q for q in range(len(segments)) if k0 <= cum[q] < k1]
            if len(mine) > 1:
                assert b == g1 + right


def check_image_windows(w, segments, cum, W, hop, cs):
    fpc = max(1, cs // hop)
    for k0, k1, a, b in w:
        s = int(np.searchsorted(cum, k0, side="right")) - 1
        if k1 <= cum[s + 1]:   # within one segment (a run of its frames, or all of them): exactly what the frames read
            st, ln = segments[s]
            f0, f1 = k0 - cum[s], k1 - cum[s]
            assert (a, b) == (st + f0 * hop, st + min(ln, (f1 - 1) * hop + W)), (k0, k1, a, b)
            assert k1 - k0 <= fpc
            continue
        mine = [q for q in range(len(segments)) if k0 <= cum[q] < k1]
        assert cum[mine[-1] + 1] == k1                                     # whole segments
        assert (a, b) == (min(segments[q][0] for q in mine), max(segments[q][0] + segments[q][1] for q in mine))
        assert b - a <= cs and k1 - k0 <= fpc
    # every input slot and output slot fits the sizes the footprint budgets
    assert ((w[:, 3] - w[:, 2]) <= max(cs, (fpc - 1) * hop + W)).all()
    assert ((w[:, 1] - w[:, 0]) <= fpc).all()


@pytest.mark.parametrize("W,hop", [(1024, 512), (1000, 500), (128, 100)])
@pytest.mark.parametrize("extra", [1, 116, 117, 511, 512, 600, 3615])
def test_image_segment_slightly_longer_than_a_chunk(L, W, hop, extra):
    """one segment a little longer than a chunk whose frames still fit one chunk: the chunk uploads only what the frames read, which
    ends before the segment whenever (len - W) % hop != 0"""
    cs = 1 << 14
    ln = cs + extra
    n = ln + 2000
    for segments in ([(1000, ln)], [(0, 999), (999, ln), (999 + ln, n - 999 - ln)]):
        frames = [num_frames(x, W, hop) for _, x in segments]
        cum = np.concatenate([[0], np.cumsum(frames)])
        w = windows(L, L.FILTER_IMAGES, n, 0, W, hop, cs, segments)
        covers_once(w, int(cum[-1]))
        check_image_windows(w, segments, cum, W, hop, cs)


def test_windows_reject_bad_arguments(L):
    lib = L.load_library()
    count = C.c_int64(0)
    assert lib.urh_stream_windows(L.FILTER_CONVOLVE, 100, 100, 0, 0, 10, None, None, 0, None, 0, C.byref(count)) != 0   # no taps
    assert lib.urh_stream_windows(L.FILTER_DB, 100, 3, 64, 0, 10, None, None, 0, None, 0, C.byref(count)) != 0         # hop 0
    assert lib.urh_stream_windows(9, 100, 100, 1, 0, 10, None, None, 0, None, 0, C.byref(count)) != 0
    st, ln = np.array([90], np.int64), np.array([20], np.int64)                                                      # past the end
    assert lib.urh_stream_windows(L.FILTER_IMAGES, 100, 0, 16, 8, 10, st.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), 1,
                                  None, 0, C.byref(count)) != 0


# ---- the schedule ---------------------------------------------------------------------------------------------------------------------
def schedule(L, win, ring, flags):
    lib = L.load_library()
    count = C.c_int64(0)
    win = np.ascontiguousarray(win, dtype=np.int64)
    assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), len(win), ring, flags, None, 0, C.byref(count)) == 0
    ops = np.zeros((max(count.value, 1), 7), np.int64)
    assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), len(win), ring, flags, ops.ctypes.data_as(C.c_void_p),
                                          count.value, C.byref(count)) == 0
    return ops[: count.value]


def _happens_before(ops, up, down):
    """edges of the model: program order per stream, and event waits resolved to the last record issued before the wait"""
    stream_of = {0: "copy0", 1: "compute", 2: "copy1"}
    last_on_stream, last_record = {}, {}
    edges = {i: set() for i in range(len(ops))}
    for i, (kind, c, s, *_rest) in enumerate(ops):
        st = stream_of[kind]
        if st in last_on_stream:
            edges[i].add(last_on_stream[st])
        waits = {0: [1], 1: ([0] if up else []) + ([2] if down else []), 2: [1]}[kind]
        for wt in waits:
            if (wt, s) in last_record:
                edges[i].add(last_record[(wt, s)])
        last_on_stream[st] = i
        last_record[(kind, s)] = i
    memo = {}

    def before(i):
        if i not in memo:
            acc = set()
            for j in edges[i]:
                acc.add(j)
                acc |= before(j)
            memo[i] = acc
        return memo[i]

    return before


@pytest.mark.parametrize("ring", [2, 3, 4])
@pytest.mark.parametrize("chunks", [1, 2, 3, 4, 5, 9])
@pytest.mark.parametrize("up,down,plan", [(True, True, "convolve"), (True, False, "convolve"), (True, True, "tiles"), (True, False, "tiles")],
                         ids=["True-True", "True-False", "tiles-True-True", "tiles-True-False"])
def test_no_slot_overwritten_before_its_readers(L, ring, chunks, up, down, plan):
    if plan == "tiles":   # whole tiles, every later chunk with the sample before it (its halo is part of its own upload)
        n = chunks * 3 * TILE - 5
        win = windows(L, L.FILTER_TILES, n, n, 1, 0, 3 * TILE)
    else:
        n, m = chunks * CS - 7, 301
        win = windows(L, L.FILTER_CONVOLVE, n, n, m, (m - 1) // 2, CS)
    assert len(win) == chunks
    flags = (L.STREAM_UPLOAD if up else 0) | (L.STREAM_DOWNLOAD if down else 0)
    ops = schedule(L, win, ring, flags)
    before = _happens_before(ops, up, down)
    idx = {(int(k), int(c)): i for i, (k, c, *_r) in enumerate(ops)}
    assert len(idx) == len(ops)
    for i, o in enumerate(ops):
        assert np.array_equal(o[3:], win[o[1]])          # every op carries its chunk's window
        assert o[2] == o[1] % ring
    for c in range(chunks):
        assert idx[(0, c)] in before(idx[(1, c)])        # the computation reads its own upload
        last_upload = max(i for i, o in enumerate(ops[: idx[(1, c)]]) if o[0] == 0 and o[2] == c % ring)
        assert ops[last_upload][1] == c                  # and no later upload into its slot came first
        for c2 in range(c % ring, c, ring):              # an upload waits for every earlier reader of its slot
            assert idx[(1, c2)] in before(idx[(0, c)])
        if down:
            assert idx[(1, c)] in before(idx[(2, c)])
            for c2 in range(c % ring, c, ring):          # the output slot is downloaded before it is rewritten
                assert idx[(2, c2)] in before(idx[(1, c)])


def test_schedule_rejects_bad_rings(L):
    lib = L.load_library()
    count = C.c_int64(0)
    win = np.zeros((2, 4), np.int64)
    for ring in (0, 1, 9):
        assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), 2, ring, 3, None, 0, C.byref(count)) != 0


# ---- footprints and the path choice ------------------------------------------------------------------------------------------------------
def fp(L, entry, n, out_len, dtype, p0, p1, cs, ring, resident):
    from urh_b200.cythonext import signal_functions as sf

    return sf.filter_footprint(entry, n, out_len, dtype, p0, p1, cs, ring, resident, cmap_entries=cmap_of(L, entry))


def cmap_of(L, entry):
    return 256 if entry == L.FILTER_IMAGES else 0


def _entries(L):
    # (entry, dtype, p0, p1, out_len(n))
    return [
        (L.FILTER_CONVOLVE, np.float32, 101, 50, lambda n: n),
        (L.FILTER_CONVOLVE, np.float32, 4001, 2000, lambda n: n),
        (L.FILTER_FIR, np.float32, 10, 0, lambda n: n),
        (L.FILTER_DC, np.float32, 0, 0, lambda n: n),
        (L.FILTER_DC, np.int16, 0, 0, lambda n: n),
        (L.FILTER_DC, np.uint8, 0, 0, lambda n: n),
        (L.FILTER_STFT, np.float32, 1024, 512, lambda n: num_frames(n, 1024, 512)),
        (L.FILTER_DB, np.float32, 1000, 700, lambda n: num_frames(n, 1000, 700)),
        (L.FILTER_IMAGES, np.float32, 1024, 512, lambda n: num_frames(n, 1024, 512) + 1000),
    ]


@pytest.mark.parametrize("k", range(9))
def test_streamed_footprint_does_not_grow_with_n(L, k):
    entry, dtype, p0, p1, out_len = _entries(L)[k]
    cs = 1 << 20
    ns = (cs + 5000, 10 * cs + 3, 1 << 30, 1 << 34)
    got = {fp(L, entry, n, out_len(n), dtype, p0, p1, cs, 2, False) for n in ns}
    assert len(got) == 1, got
    res = [fp(L, entry, n, out_len(n), dtype, p0, p1, cs, 2, True) for n in ns]
    assert all(a < b for a, b in zip(res, res[1:]))
    assert got.pop() < res[-1] / 100


@pytest.mark.parametrize("k", range(9))
def test_path_choice_at_the_budget(L, k):
    from urh_b200.cythonext import signal_functions as sf

    entry, dtype, p0, p1, out_len = _entries(L)[k]
    for n in (5000, 1 << 22, 1 << 31):
        c = cmap_of(L, entry)
        need = sf.filter_footprint(entry, n, out_len(n), dtype, p0, p1, resident=True, cmap_entries=c)
        assert sf.filter_use_stream(entry, n, out_len(n), dtype, p0, p1, need - 1, cmap_entries=c)
        assert not sf.filter_use_stream(entry, n, out_len(n), dtype, p0, p1, need, cmap_entries=c)


@pytest.mark.parametrize("resident", [False, True])
def test_image_footprint_counts_the_colormap(L, resident):
    from urh_b200.cythonext import signal_functions as sf

    n = 1 << 26
    f = [sf.filter_footprint(L.FILTER_IMAGES, n, num_frames(n, 1024, 512), np.float32, 1024, 512, 1 << 20, 2, resident, cmap_entries=e)
         for e in (256, 1 << 16, 1 << 20)]
    assert f[1] - f[0] == 4 * ((1 << 16) - 256) and f[2] - f[1] == 4 * ((1 << 20) - (1 << 16))


def test_footprint_rejects_bad_arguments(L):
    lib = L.load_library()
    out = C.c_int64(0)
    assert lib.urh_stream_filter_footprint(L.FILTER_CONVOLVE, 100, 100, L.DT_F32, 0, 0, 0, 10, 2, 0, C.byref(out)) != 0
    assert lib.urh_stream_filter_footprint(L.FILTER_DB, 100, 3, L.DT_F32, 64, 32, 0, 10, 1, 0, C.byref(out)) != 0
    assert lib.urh_stream_filter_footprint(L.FILTER_DC, 100, 100, 17, 0, 0, 0, 10, 2, 0, C.byref(out)) != 0
    assert lib.urh_stream_filter_footprint(6, 100, 100, L.DT_F32, 1, 0, 0, 10, 2, 0, C.byref(out)) != 0
    assert lib.urh_stream_filter_footprint(L.FILTER_IMAGES, 100, 3, L.DT_F32, 64, 32, 0, 10, 2, 0, C.byref(out)) != 0   # no colormap
