"""CPU suite: the host plans of the sharded band-pass / FIR / DC correction / spectrogram (urh_b200/dist.py) against float64 models
of the whole capture.  Samples and taps are small integers, so every product and sum below is exact and an off-by-one halo or
offset shows up as an exact mismatch, not as rounding noise."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from urh_b200 import dist as udist  # noqa: E402


def random_bounds(rng, n, world, min_len=1):
    """contiguous shards of random, unequal, unaligned lengths >= min_len (n >= world * min_len)"""
    extra = n - world * min_len
    cuts = np.sort(rng.integers(0, extra + 1, world - 1))
    lengths = np.diff(np.concatenate([[0], cuts, [extra]])) + min_len
    edges = np.concatenate([[0], np.cumsum(lengths)]).astype(int)
    return [(int(edges[i]), int(edges[i + 1])) for i in range(world)]


def tight_bounds(n, world, halo):
    """every shard but the last exactly `halo` samples long"""
    edges = [r * halo for r in range(world)] + [n]
    return [(edges[i], edges[i + 1]) for i in range(world)]


def int_signal(rng, n):
    return (rng.integers(-8, 9, n) + 1j * rng.integers(-8, 9, n)).astype(np.complex128)


def int_taps(rng, m):
    return (rng.integers(-4, 5, m) + 1j * rng.integers(-4, 5, m)).astype(np.complex128)


def valid_bounds(plan_fn, rng, n, world, min_len):
    for _ in range(50):
        b = random_bounds(rng, n, world, min_len)
        try:
            return b, plan_fn(b)
        except ValueError:
            continue
    raise AssertionError("no valid bounds drawn")


@pytest.mark.parametrize("m", [1, 3, 11, 41, 101, 401])
def test_bandpass_plan_model_equals_whole_capture(m):
    rng = np.random.default_rng(m)
    for trial in range(12):
        world = int(rng.integers(2, 9))
        n = int(rng.integers(max(m, 8) * world, max(m, 8) * world * 5))
        half = (m - 1) // 2
        if trial % 3 == 0:
            bounds = tight_bounds(n, world, max(half, m - 1 - half, 1))
            plan = udist.bandpass_plan(n, m, bounds)
        else:
            bounds, plan = valid_bounds(lambda b: udist.bandpass_plan(n, m, b), rng, n, world, max(half, 1))
        x, h = int_signal(rng, n), int_taps(rng, m)
        parts = []
        for (g0, g1), (left, right, offset) in zip(bounds, plan):
            win = x[g0 - left: g1 + right]
            parts.append(np.convolve(win, h)[offset: offset + (g1 - g0)])
        got = np.concatenate(parts)
        assert np.array_equal(got, np.convolve(x, h, "same")), (m, bounds)
        # the FFT branch's centred crop of the full convolution (Filter.fft_convolve_1d) is the same slice for an odd filter
        too_much = (n + m - 1 - n) // 2
        if too_much:
            assert np.array_equal(got, np.convolve(x, h)[too_much: n + m - 1 - too_much])


@pytest.mark.parametrize("m", [0, 1, 2, 10, 101, 1000])
def test_fir_plan_model_equals_serial_fir(m):
    rng = np.random.default_rng(100 + m)
    for trial in range(12):
        world = int(rng.integers(2, 9))
        n = int(rng.integers(max(m, 4) * world, max(m, 4) * world * 4))
        if trial % 3 == 0:
            bounds = tight_bounds(n, world, max(m - 1, 1))
            hist = udist.fir_plan(n, m, bounds)
        else:
            bounds, hist = valid_bounds(lambda b: udist.fir_plan(n, m, b), rng, n, world, max(m - 1, 1))
        x, taps = int_signal(rng, n), int_taps(rng, m)
        # the reference's serial fir_filter: y[k] = sum over i ascending of x[i] * taps[k - i]
        ref = np.convolve(x, taps)[:n] if m else np.zeros(n, np.complex128)
        parts = []
        for (g0, g1), h in zip(bounds, hist):
            win = x[g0 - h: g1]
            parts.append(np.convolve(win, taps)[h: h + (g1 - g0)] if m else np.zeros(g1 - g0, np.complex128))
        assert np.array_equal(np.concatenate(parts), ref), (m, bounds)


@pytest.mark.parametrize("W,overlap", [(1024, 0.5), (256, 0.75), (1000, 0.5), (128, 0.0), (64, 0.9)])
def test_frame_plan_owns_every_frame_once_inside_the_window(W, overlap):
    rng = np.random.default_rng(W)
    hop = W - int(overlap * W)
    for trial in range(40):
        world = int(rng.integers(1, 9))
        n = int(rng.integers(max(1, W // 3), W * 60))
        try:
            bounds = random_bounds(rng, n, world, 1) if n >= world else [(0, n)]
            plan = udist.frame_plan(n, W, hop, bounds)
        except ValueError:
            continue   # a shard shorter than the tail a frame needs from it
        frames = max(1, (max(n, W) - W) // hop + 1)
        owned = [f for f0, nf, _ in plan for f in range(f0, f0 + nf)]
        assert owned == list(range(frames))
        for (g0, g1), (f0, nf, right) in zip(bounds, plan):
            for f in range(f0, f0 + nf):
                assert g0 <= f * hop < g1                       # owned by the rank holding its first sample
                assert min(n, f * hop + W) <= g1 + right         # every sample it reads is in the extended window
            assert right <= W - 1


def test_frame_plan_edges_not_multiples_of_hop():
    n, W, hop = 10_000, 1024, 512
    bounds = [(0, 3000), (3000, 7001), (7001, n)]
    assert udist.frame_plan(n, W, hop, bounds) == [(0, 6, 584), (6, 8, 679), (14, 4, 0)]


@pytest.mark.parametrize("W,overlap,max_lines", [(1024, 0.5, 1000), (256, 0.75, 7), (100, 0.5, 3), (64, 0.0, 50)])
def test_segment_plan_equals_segment_bounds(W, overlap, max_lines):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    rng = np.random.default_rng(W + max_lines)
    for trial in range(20):
        n = int(rng.integers(W, W * 400))
        world = int(rng.integers(1, 6))
        spec = Spectrogram(np.zeros(n, np.complex64), window_size=W, overlap_factor=overlap)
        spec.MAX_LINES_PER_VIEW = max_lines
        try:
            bounds = random_bounds(rng, n, world, 1)
            segments, owned, rights = udist.segment_plan(n, W, spec.hop_size, bounds, max_lines)
        except ValueError:
            continue
        assert segments == spec.segment_bounds()
        assert [i for mine in owned for i in mine] == list(range(len(segments)))
        for (g0, g1), mine, right in zip(bounds, owned, rights):
            for i in mine:
                s, e, _ = segments[i]
                assert g0 <= s < g1 and e <= g1 + right


def test_plans_validate():
    # the single-GPU band-pass changes the length (N < M) or returns nothing (M <= 2 on the FFT branch)
    with pytest.raises(ValueError, match="shorter than the 101-tap filter"):
        udist.bandpass_plan(100, 101, [(0, 50), (50, 100)])
    with pytest.raises(ValueError, match="empty array"):
        udist.bandpass_plan(1, 1, [(0, 1)])
    with pytest.raises(ValueError, match="even"):
        udist.bandpass_plan(10, 10, [(0, 5), (5, 10)])
    # a shard shorter than the halo it must supply
    with pytest.raises(ValueError, match="shorter than the 50-sample halo"):
        udist.bandpass_plan(1000, 101, [(0, 49), (49, 1000)])
    with pytest.raises(ValueError, match="shorter than the 50-sample halo"):
        udist.bandpass_plan(1000, 101, [(0, 900), (900, 949), (949, 1000)])
    with pytest.raises(ValueError, match="shorter than the 9-sample halo"):
        udist.fir_plan(100, 10, [(0, 8), (8, 100)])
    with pytest.raises(ValueError, match="spectrogram"):
        udist.frame_plan(10_000, 1024, 512, [(0, 9_000), (9_000, 9_010), (9_010, 10_000)])
    with pytest.raises(ValueError, match="bounds"):
        udist.fir_plan(100, 10, [(0, 50), (60, 100)])
    with pytest.raises(ValueError, match="bounds"):
        udist.fir_plan(100, 10, [(0, 50), (50, 50), (50, 100)])
    # exactly one halo long is enough
    assert udist.bandpass_plan(1000, 101, [(0, 50), (50, 100), (100, 1000)])[1] == (50, 50, 100)
    assert udist.fir_plan(100, 10, [(0, 9), (9, 100)]) == [0, 9]


def test_dc_fold_double_rank_order():
    parts = np.array([[1e16, 3.0], [1.0, -3.0], [-1e16, 1.5]])
    s = (1e16 + 1.0) + -1e16, (3.0 + -3.0) + 1.5
    assert np.array_equal(udist.dc_fold_double(parts, 3), (np.array(s) / 3.0).astype(np.float32))


def _dc_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    from urh_b200.dist import HostExchange, dc_exact_handover, bandpass_plan, frame_plan

    hx = HostExchange()
    ok = True
    for trial, n in enumerate([1, 2, 1023, 100_003, 3 * 2 ** 15 + 5]):
        rng = np.random.default_rng(7 + trial)   # same capture on every rank
        x = (rng.standard_normal((n, 2)) * 3 + 0.25).astype(np.float32)
        cut = int(rng.integers(0, n + 1))
        lo, hi = [(0, cut), (cut, n)][rank]

        def chain(carry):
            cols = np.concatenate([np.asarray(carry, np.float32)[None, :], x[lo:hi]])
            return np.add.accumulate(cols, axis=0, dtype=np.float32)[-1]

        got = dc_exact_handover(rank, world, chain, lambda v: np.stack(hx.allgather(np.asarray(v, np.float32))))
        ref = np.sum(x, axis=0, dtype=np.float32)   # what np.mean(x, axis=0) divides: the serial row-order chain
        ok = ok and got.dtype == np.float32 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
        ok = ok and np.array_equal((got / np.float32(n)).view(np.uint32), np.mean(x, axis=0).view(np.uint32))
    # every rank raises the same error, before any collective
    for fn in (lambda: bandpass_plan(100, 101, [(0, 50), (50, 100)]), lambda: frame_plan(10_000, 1024, 512, [(0, 9_000), (9_000, 9_010), (9_010, 10_000)])):
        try:
            fn()
            msg = None
        except ValueError as e:
            msg = str(e)
        msgs = hx.allgather(msg)
        ok = ok and msg is not None and all(m == msgs[0] for m in msgs)
    res = hx.allgather(bool(ok))
    if rank == 0:
        open(os.path.join(tmp, "ok"), "w").write("1" if all(res) else "0")
    dist.destroy_process_group()


def test_dc_exact_handover_gloo(tmp_path):
    import torch.multiprocessing as mp

    port = 29870 + os.getpid() % 100
    mp.spawn(_dc_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert open(tmp_path / "ok").read() == "1"

