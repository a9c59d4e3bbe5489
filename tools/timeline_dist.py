#!/usr/bin/env python
"""Where a sharded step spends its time between GPUs: per-rank stream timeline of urh_shard_demod_center_digitize on bench.py's
capture (N x 2^log2n samples sharded over N GPUs), from CUDA events the library records at the step's start, on either side of
every inter-GPU exchange and after the rows are written (urh_set_profiling(ctx, 2) / urh_timeline_fetch).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/timeline_dist.py --log2n 30

Steps run back to back without a barrier, as in bench.py (the last exchange of a step leaves the ranks aligned).  Reading the output:
a COMPUTE segment (exchange done -> next exchange enter) is this rank's own kernels, so its spread over the ranks is the GPUs'
speed spread; an EXCHANGE segment (enter -> done) is the collective's latency plus the wait for the slowest rank, so its MINIMUM
over the ranks is the exchange's own cost and the rest is skew.  One JSON line on rank 0."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--global-gaps", action="store_true",
                    help="long gap / tail defined on the whole capture (round-2 measurement of the load imbalance) instead of per block")
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    if world < 2:
        sys.exit("run under torchrun with at least 2 ranks")
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    import bench as B
    from urh_b200 import _lib, dist as udist
    from urh_b200.device import DeviceArray

    ctx = _lib.default_context(local_rank)
    lib = ctx.lib
    n = 1 << args.log2n
    n_total, offset = n * world, n * rank
    nsym = n // B.SPS + 2
    b, s = B.make_symbols(nsym, seed=1000 + rank)
    d_b = DeviceArray(ctx, (nsym,), np.int8).set(b)
    d_s = DeviceArray(ctx, (nsym,), np.int32).set(s)
    sb = udist.ShardBuffer(ctx, n, np.float32)
    d_qad = DeviceArray(ctx, (n,), np.float32)
    ctx.check(lib.urh_synth_fsk(ctx.handle, C.c_void_p(sb.shard.ptr), n, offset, B.SPS, C.c_void_p(d_b.ptr), C.c_void_p(d_s.ptr),
                                C.c_double(B.FDEV / B.FS), 1.0, B.SIGMA, 12345, 6_000_000, 5_000_000,
                                *(B.capture_gaps(n, rank) if not args.global_gaps else
                                  (int(0.40 * n_total), int(0.43 * n_total), int(0.97 * n_total)))))
    ctx.sync()
    hx = udist.HostExchange()
    udist.init_nccl(ctx, hx)
    udist.exchange_halo(ctx, hx, sb)

    def step():
        return udist.demod_center_digitize_distributed(ctx, rank, world, sb, offset, n_total, B.NOISE_MAG, "FSK", B.TOL, B.SPS, d_qad,
                                                       fetch=False)

    lib.urh_set_profiling(ctx.handle, 2)
    for _ in range(args.warmup):
        step()
    ctx.sync()
    dist.barrier()
    marks, names = [], None
    ms = (C.c_float * 32)()
    buf = C.create_string_buffer(2048)
    cnt = C.c_int(0)
    for _ in range(args.steps):
        step()
        ctx.check(lib.urh_timeline_fetch(ctx.handle, ms, buf, 2048, C.byref(cnt)))
        marks.append([ms[i] for i in range(cnt.value)])
        names = buf.value.decode().strip().split("\n")
    mine = np.median(np.array(marks), axis=0)   # this rank's median time of each mark
    every = [None] * world
    dist.all_gather_object(every, [float(x) for x in mine])
    if rank == 0:
        t = np.array(every)                     # [rank, mark], ms since the rank's own step start
        seg = np.diff(t, axis=1) * 1e3          # us per segment
        rows = []
        for i in range(seg.shape[1]):
            kind = "exchange" if names[i].endswith("enter") else "compute"
            rows.append({"from": names[i], "to": names[i + 1], "kind": kind, "us_min": float(seg[:, i].min()),
                         "us_median": float(np.median(seg[:, i])), "us_max": float(seg[:, i].max())})
        compute_max = sum(r["us_max"] for r in rows if r["kind"] == "compute")
        compute_med = sum(r["us_median"] for r in rows if r["kind"] == "compute")
        exch_min = sum(r["us_min"] for r in rows if r["kind"] == "exchange")
        exch_med = sum(r["us_median"] for r in rows if r["kind"] == "exchange")
        print(json.dumps({
            "what": "stream timeline of the sharded step (demod + detect_center + digitize), %d x 2^%d samples on %d GPUs, median of %d steps"
                    % (world, args.log2n, world, args.steps),
            "exchange": "NCCL",
            "segments": rows,
            "step_us_median_over_ranks": float(np.median(t[:, -1]) * 1e3),
            "sum_compute_us": {"median_rank": compute_med, "slowest_rank_per_segment": compute_max},
            "sum_exchange_us": {"median_rank": exch_med, "fastest_rank_per_exchange (= the exchanges' own cost)": exch_min},
            "per_rank_first_compute_segment_us (demodulation: the GPUs' speed spread)": [float(x) for x in seg[:, 0]],
        }))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
