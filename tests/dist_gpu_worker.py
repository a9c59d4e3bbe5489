"""Worker for tests/test_gpu_dist.py: launched under torchrun with one rank per GPU.  Compares the sharded
demod+digitize / noise detection (urh_b200.dist, NCCL) with the single-GPU result on the same capture."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch.distributed as dist

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from conftest import synth_fsk
    from urh_b200 import _lib, dist as udist
    from urh_b200.device import DeviceArray
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.ainterpretation import AutoInterpretation as AI

    ctx = _lib.default_context(int(os.environ.get("LOCAL_RANK", rank)))
    hx = udist.HostExchange()
    udist.init_nccl(ctx, hx)
    failures = []
    for case, (n, sps, tol, mod, dtype) in enumerate([
        (3_000_000, 100, 5, "FSK", np.float32), (1_000_003, 37, 0, "FSK", np.float32), (700_001, 50, 9, "ASK", np.float32),
        (2_500_000, 100, 5000, "FSK", np.float32), (900_000, 64, 3, "FSK", np.int16),
    ]):
        iq = synth_fsk(n, sps=sps, seed=17 + case, gap_every=n // 7, dtype=dtype)
        if mod == "ASK":
            env = np.repeat(np.random.default_rng(case).integers(0, 2, n // sps + 1), sps)[:n] * 0.9 + 0.1
            iq = (iq.astype(np.float32) * env[:, None]).astype(dtype)
        noise = 0.05 if dtype == np.float32 else 1000.0
        center = 0.0 if mod == "FSK" else 0.3
        lo, hi = udist.shard_bounds(n, world)[rank]
        sb = udist.ShardBuffer(ctx, hi - lo, dtype)
        sb.shard.set(iq[lo:hi])
        udist.exchange_halo(ctx, hx, sb)
        d_qad = DeviceArray(ctx, (hi - lo,), np.float32)
        part = udist.demod_digitize_distributed(ctx, rank, world, sb, lo, n, noise, mod, center, tol, sps, d_qad=d_qad)
        qads = hx.allgather(d_qad.get())
        parts = hx.allgather(part)
        noise_sh = udist.detect_noise_level_sharded(ctx, hx, sb, lo, n)
        d_qad2 = DeviceArray(ctx, (hi - lo,), np.float32)
        c_sh, part_c = udist.demod_center_digitize_distributed(ctx, rank, world, sb, lo, n, noise, mod, tol, sps, d_qad2)
        parts_c = hx.allgather(part_c)
        centers = hx.allgather(c_sh)
        if rank == 0:
            qad_ref, rows_ref = sf.demod_digitize(iq, noise, mod, center, tol, sps)
            if not np.array_equal(np.concatenate(qads).view(np.uint32), qad_ref.view(np.uint32)):
                failures.append(("qad", case))
            rows = udist.merge_shard_rows(parts)
            if not np.array_equal(rows, rows_ref):
                failures.append(("rows", case, len(rows), len(rows_ref)))
            if noise_sh != AI.detect_noise_level_iq(iq):
                failures.append(("noise", case, noise_sh))
            c_one, rows_one = sf.demod_center_digitize(iq, noise, mod, tol, sps)
            if any(c != centers[0] for c in centers):
                failures.append(("center differs between ranks", case, centers))
            if (c_one is None) != (c_sh is None) or (c_one is not None and abs(c_one - c_sh) > 1e-9 * max(1.0, abs(c_one))):
                failures.append(("center", case, c_sh, c_one))
            elif c_one is not None and not np.array_equal(udist.merge_shard_rows(parts_c), sf.grab_pulse_lens(qad_ref, c_sh, tol, mod, sps)):
                failures.append(("rows_center", case))
    # PSK: speculative Costas loop over shards == single-GPU == oracle (bit-exact)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_costas import synth_psk

    for order in (2, 4):
        n = 1_200_000
        iq = synth_psk(n, order, seed=40 + order, gap_period=250000, gap_len=60000)
        lo, hi = udist.shard_bounds(n, world)[rank]
        sb = udist.ShardBuffer(ctx, hi - lo, np.float32, halo=udist.costas_halo(ctx))
        sb.shard.set(iq[lo:hi])
        udist.exchange_halo(ctx, hx, sb)
        d_out = DeviceArray(ctx, (hi - lo,), np.float32)
        udist.afp_demod_psk_sharded(ctx, rank, world, sb, 0.2, order, 0.1, d_out)
        parts = hx.allgather(d_out.get())
        if rank == 0:
            ref = sf.afp_demod(iq, 0.2, "PSK", order)
            got = np.concatenate(parts)
            if not np.array_equal(got[1:].view(np.uint32), ref[1:].view(np.uint32)):
                failures.append(("psk", order, int((got[1:].view(np.uint32) != ref[1:].view(np.uint32)).sum())))
    # AutoInterpretation.estimate over shards == estimate on one GPU (BASELINE configs[4] shape, small)
    from urh_b200.signalprocessing.IQArray import IQArray
    for kind in ("FSK", "PSK"):
        n = 2_400_000
        if kind == "FSK":
            iq = synth_fsk(n, sps=100, seed=91, gap_every=150_000)
            iq[-60_000:] *= 0.001
        else:
            iq = synth_psk(n, 2, seed=92, gap_period=300_000, gap_len=90_000)
        bounds = udist.shard_bounds(n, world)
        lo, hi = bounds[rank]
        sb = udist.ShardBuffer(ctx, hi - lo, np.float32, halo=udist.costas_halo(ctx))
        sb.shard.set(iq[lo:hi])
        udist.exchange_halo(ctx, hx, sb)
        for given in (kind, None):
            est = udist.estimate_sharded(ctx, hx, sb, bounds, n, noise=None, modulation=given)
            ests = hx.allgather(est)
            if rank == 0:
                one = AI.estimate(IQArray(iq), noise=None, modulation=given)
                if any(e != ests[0] for e in ests):
                    failures.append(("estimate differs between ranks", kind, given))
                if one != est:
                    failures.append(("estimate", kind, given, est, one))
    res = hx.allgather(failures)
    if rank == 0:
        flat = [f for part in res for f in part]
        print("DIST_GPU_RESULT", "OK" if not flat else flat)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
