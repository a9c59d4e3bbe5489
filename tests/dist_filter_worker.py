"""Worker for tests/test_gpu_dist_filter.py: launched under torchrun with one rank per GPU.  Every sharded result is gathered on rank 0
and compared bit for bit with the single-GPU public function on the whole capture."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def capture(n, seed, dtype=np.float32):
    rng = np.random.default_rng(seed)
    if dtype != np.float32:
        info = np.iinfo(dtype)
        return rng.integers(info.min, info.max + 1, (n, 2)).astype(dtype)
    t = np.arange(n)
    x = np.exp(2j * np.pi * 0.05 * t) * (1 + 0.5 * (rng.random(n) > 0.5)) + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    x += 0.3 - 0.2j
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))


def uneven_bounds(n, world, seed):
    """contiguous shards of unequal lengths whose edges are not multiples of any hop"""
    rng = np.random.default_rng(seed)
    w = rng.random(world) + 0.5
    edges = np.concatenate([[0], np.floor(np.cumsum(w) / w.sum() * n)]).astype(np.int64)
    edges[-1] = n
    edges[1:-1] += 1 - edges[1:-1] % 2   # odd edges
    return [(int(edges[i]), int(edges[i + 1])) for i in range(world)]


def main():
    import torch.distributed as dist

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from urh_b200 import _lib, dist as udist
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Filter import Filter, FilterType
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    ctx = _lib.default_context(int(os.environ.get("LOCAL_RANK", rank)))
    hx = udist.HostExchange()
    udist.init_nccl(ctx, hx)
    failures = []

    def shard(x, bounds, halo=1):
        lo, hi = bounds[rank]
        sb = udist.ShardBuffer(ctx, hi - lo, x.dtype, halo=halo)
        sb.shard.set(x[lo:hi])
        return sb

    def gathered(arr):
        parts = hx.allgather(arr)
        return np.concatenate(parts) if rank == 0 else None

    def same(a, b):
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))

    # ---- band-pass at every bandwidth preset and 101 taps, swapped and clipped edges
    n = 1_000_003
    x = capture(n, 1)
    xc = x.view(np.complex64).reshape(-1)
    bounds = uneven_bounds(n, world, 1)
    sb = shard(x, bounds)
    cases = [(0.03, 0.07, bw) for bw in Filter.BANDWIDTHS.values()] + [(0.07, 0.03, Filter.get_bandwidth_from_filter_length(101)),
                                                                      (-0.8, 0.1, 0.08)]
    for f_low, f_high, bw in cases:
        out = udist.apply_bandpass_filter_sharded(ctx, hx, sb, bounds, f_low, f_high, bw)
        got = gathered(out.shard.get())
        # the output's left halo holds the previous shard's filtered tail
        halos = hx.allgather(out.halo.get() if rank else None)
        if rank == 0:
            ref = Filter.apply_bandpass_filter(xc, f_low, f_high, bw).view(np.float32).reshape(-1, 2)
            if not same(got, ref):
                failures.append(("band-pass", f_low, f_high, bw, int((got != ref).any(axis=1).sum())))
            for r in range(1, world):
                g0 = bounds[r][0]
                if not same(halos[r], ref[g0 - out.halo_len: g0]):
                    failures.append(("band-pass output halo", bw, r))
    # ---- the band-passed chain: ASK demod + center + digitize over the filtered shards
    env = np.repeat(np.random.default_rng(9).integers(0, 2, n // 200 + 1), 200)[:n] * 0.9 + 0.1
    xa = np.ascontiguousarray((x * env[:, None]).astype(np.float32))
    sba = shard(xa, bounds)
    filt = udist.apply_bandpass_filter_sharded(ctx, hx, sba, bounds, 0.03, 0.07, Filter.get_bandwidth_from_filter_length(101))
    from urh_b200.device import DeviceArray
    d_qad = DeviceArray(ctx, (filt.n,), np.float32)
    center, part = udist.demod_center_digitize_distributed(ctx, rank, world, filt, bounds[rank][0], n, 0.05, "ASK", 5, 200, d_qad)
    parts = hx.allgather(part)
    centers = hx.allgather(center)
    if rank == 0:
        one = Filter.apply_bandpass_filter(xa.view(np.complex64).reshape(-1), 0.03, 0.07, Filter.get_bandwidth_from_filter_length(101))
        c_one, rows_one = sf.demod_center_digitize(np.ascontiguousarray(one.view(np.float32).reshape(-1, 2)), 0.05, "ASK", 5, 200)
        if any(c != centers[0] for c in centers) or c_one != center:
            failures.append(("band-passed chain center", centers, c_one))
        elif not np.array_equal(udist.merge_shard_rows(parts), rows_one):
            failures.append(("band-passed chain rows",))
    # ---- FIR with 1, 10, 101 taps (Filter.work)
    for m in (1, 10, 101):
        taps = list((np.random.default_rng(m).standard_normal(m) / m).astype(np.complex64))
        out = udist.filter_work_sharded(ctx, hx, sb, bounds, Filter(taps, FilterType.custom))
        got = gathered(out.shard.get())
        if rank == 0 and not same(got, Filter(taps).work(x).view(np.float32).reshape(-1, 2)):
            failures.append(("fir", m))
    # ---- DC correction: float32 in both regimes, int8 and int16
    for nd, dtype in [(3 * 2 ** 20 + 5, np.float32), (5_000_000, np.float32), (1_000_001, np.int8), (999_999, np.int16)]:
        xd = capture(nd, nd, dtype)
        bd = uneven_bounds(nd, world, nd)
        out = udist.filter_work_sharded(ctx, hx, shard(xd, bd), bd, Filter([0.1], FilterType.dc_correction))
        got = gathered(out.shard.get())
        if rank == 0:
            if dtype == np.float32 and nd > Filter.EXACT_DC_MAX:
                ref = xd - np.mean(xd.astype(np.float64), axis=0).astype(np.float32)
            else:
                ref = Filter.dc_correction(xd)
            if not same(got, ref):
                failures.append(("dc", nd, np.dtype(dtype).name))
    # ---- dB map: k_stft_r16 at 1024 / 512 and at 256 with overlap 0.75, cuFFT-composed 1000 / 500; shard edges not multiples of hop
    for W, overlap in [(1024, 0.5), (256, 0.75), (1000, 0.5)]:
        first, db = udist.spectrogram_db_sharded(ctx, hx, sb, bounds, W, overlap)
        firsts = hx.allgather(first)
        got = gathered(db.get())
        if rank == 0:
            ref = Spectrogram(xc, window_size=W, overlap_factor=overlap).calculate_spectrogram()
            if not same(got, ref) or firsts != sorted(firsts):
                failures.append(("db", W, overlap))
    # ---- images, both layouts
    cmap = np.random.default_rng(4).integers(0, 256, (256, 4)).astype(np.uint8)
    nbig = 2_500_003
    xb = capture(nbig, 5)
    bb = uneven_bounds(nbig, world, 5)
    sbb = shard(xb, bb)
    for W, overlap, transpose in [(1024, 0.5, False), (256, 0.75, True), (1024, 0.5, True)]:
        mine = udist.spectrogram_image_segments_sharded(ctx, hx, sbb, bb, W, overlap, colormap=cmap, transpose=transpose)
        every = hx.allgather([(i, img.get()) for i, img in mine])
        if rank == 0:
            got = sorted((i, img) for part in every for i, img in part)
            spec = Spectrogram(xb.view(np.complex64).reshape(-1), window_size=W, overlap_factor=overlap)
            if transpose:
                ref = [spec.create_spectrogram_image(s, e, transpose=True, colormap=cmap) for s, e, _ in spec.segment_bounds()]
            else:
                ref = list(spec.create_image_segments(colormap=cmap))
            if [i for i, _ in got] != list(range(len(ref))) or not all(same(a, b) for (_, a), b in zip(got, ref)):
                failures.append(("images", W, overlap, transpose))
    # ---- validation raises on every rank alike, before any collective
    try:
        udist.apply_bandpass_filter_sharded(ctx, hx, sb, [(0, 10), (10, n)] if world == 2 else [(0, 10)] + bounds[1:], 0.03, 0.07, 0.001)
        msg = None
    except ValueError as e:
        msg = str(e)
    msgs = hx.allgather(msg)
    if rank == 0 and (msg is None or any(m != msg for m in msgs)):
        failures.append(("validation", msgs))
    res = hx.allgather(failures)
    if rank == 0:
        flat = [f for part in res for f in part]
        print("DIST_FILTER_RESULT", "OK" if not flat else flat, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
