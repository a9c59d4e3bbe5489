#!/usr/bin/env python
"""Modulator throughput, kernel vs host: Modulator-style batches of random messages -> IQ in HBM.

    python tools/bench_modulate.py [--nmsg 10000 --bits 1000 --sps 100] > modulate.jsonl
    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file mod_launches.csv python tools/bench_modulate.py --reps 1

Per modulation: wall time of signal_functions.modulate_batch (rectangular [nmsg, nbits] input, result left in HBM), the
CUDA-event time of the library call alone (urh_modulate_batch: H2D of four offset vectors, memset of the output, the
kernels), and the host share (Python prep + upload of the bits + allocation).  Write-only roofline: 8 B/sample."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nmsg", type=int, default=10000)
    ap.add_argument("--bits", type=int, default=1000)
    ap.add_argument("--sps", type=int, default=100)
    ap.add_argument("--pause", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.cythonext import signal_functions as sf

    ctx = _lib.default_context()
    peak = 3350.0   # H100 SXM data sheet (HBM3), unless MEASURED_PEAKS.json gives a measured figure
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    rng = np.random.default_rng(2)
    bits = rng.integers(0, 2, (args.nmsg, args.bits), dtype=np.uint8)
    cases = [("ASK", [0.0, 1.0], 40e3), ("FSK", [-20e3, 20e3], 0.0), ("PSK", [np.pi / 2, -np.pi / 2], 40e3), ("GFSK", [-20e3, 20e3], 0.0)]
    for mod, params, fc in cases:
        params = np.array(params, np.float32)
        walls, devs = [], []
        total = 0
        for rep in range(args.reps + 1):
            ctx.sync()
            t0 = time.perf_counter()
            ctx.timer_start()
            d_out, off = sf.modulate_batch(bits, args.sps, mod, params, 1, 1.0, fc, 0.0, 2e6, args.pause, 0, np.float32, device_result=True)
            dev_ms = ctx.timer_stop()
            wall = (time.perf_counter() - t0) * 1e3
            total = int(off[-1])
            d_out.free()
            if rep:   # first call: allocation of the pool
                walls.append(wall)
                devs.append(dev_ms)
        wall, dev = float(np.median(walls)), float(np.median(devs))
        st = (C.c_int64 * 2)()
        ctx.lib.urh_modulate_stats(ctx.handle, st)
        print(json.dumps({"path": "modulate_batch %s %d x %d bits x %d sps + %d pause" % (mod, args.nmsg, args.bits, args.sps, args.pause),
                          "samples": total, "wall_ms": wall, "stream_ms": dev,
                          "GS_per_s_wall": total / wall / 1e6, "GS_per_s_stream": total / dev / 1e6,
                          "write_GBps_stream": 8 * total / dev / 1e6, "gfsk_phase_steps_prefix_sum_vs_serial": [int(st[0]), int(st[1])], "frac_of_hbm_peak_stream": 8 * total / dev / 1e6 / peak}), flush=True)


if __name__ == "__main__":
    main()
