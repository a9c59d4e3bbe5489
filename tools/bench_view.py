"""Time the signal view (path_creator.create_path_streams) on captures resident in HBM, and the reference's compiled create_path.

    python tools/bench_view.py [--log2n 30] [--reps 20] [--out FILE]

Scene type 0 draws one IQ column (a DeviceColumn of an (n, 2) capture: the kernel reads every other element, so both columns'
bytes cross the bus); scene type 1 draws qad (float32, contiguous).  Each is timed at full view and at a 1/64 view: the whole call up
to the bytes on the host with the host clock, and the min/max kernel alone with CUDA events.  Bytes per sample is what DRAM has
to deliver: the (n, 2) row for a column (sectors are shared), the sample itself for qad.  The reference's create_path (OpenMP
Cython, oracle/_ref/path_creator, when built) is timed on a 2^26-sample host slice with its own thread choice.  Prints one JSON
line.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from urh_b200 import _lib, settings
    from urh_b200.cythonext import path_creator as pc
    from urh_b200.device import DeviceArray, DeviceColumn

    ctx = _lib.default_context()
    n = 1 << args.log2n
    g = torch.Generator(device="cuda").manual_seed(1)
    sources = {}
    f32 = torch.randn((n, 2), device="cuda", dtype=torch.float32, generator=g)
    sources["float32 IQ column (scene 0)"] = (DeviceColumn(DeviceArray(ctx, (n, 2), np.float32, ptr=f32.data_ptr(), base=f32), 0), 8)
    i8 = torch.randint(-128, 128, (n, 2), device="cuda", dtype=torch.int8, generator=g)
    sources["int8 IQ column (scene 0)"] = (DeviceColumn(DeviceArray(ctx, (n, 2), np.int8, ptr=i8.data_ptr(), base=i8), 0), 2)
    qad = torch.randn((n,), device="cuda", dtype=torch.float32, generator=g)
    sources["qad float32 (scene 1)"] = (DeviceArray(ctx, (n,), np.float32, ptr=qad.data_ptr(), base=qad), 4)
    torch.cuda.synchronize()

    rows = []
    for name, (src, bps) in sources.items():
        for view, (a, b) in (("full", (0, n)), ("1/64", (n // 3, n // 3 + n // 64))):
            N = b - a
            spp = int(N / settings.PIXELS_PER_PATH)
            P = -(-N // spp)
            values = DeviceArray(ctx, (2 * P,), src.dtype)
            dt, stride = _lib.dtype_code(src.dtype), getattr(src, "stride", 1)
            for _ in range(3):
                pc.create_path_streams(src, a, b)
            t0 = time.perf_counter()
            for _ in range(args.reps):
                streams = pc.create_path_streams(src, a, b)
            call_ms = (time.perf_counter() - t0) * 1e3 / args.reps
            ctx.timer_start()
            for _ in range(args.reps):
                ctx.check(ctx.lib.urh_path_minmax(ctx.handle, C.c_void_p(src.ptr), dt, stride, len(src), a, b, spp, C.c_void_p(values.ptr)))
            kernel_ms = ctx.timer_stop() / args.reps
            rows.append(dict(source=name, view=view, samples=N, samples_per_pixel=spp, stream_bytes=len(streams[0]),
                             bytes_per_sample=bps, call_ms=round(call_ms, 4), minmax_kernel_ms=round(kernel_ms, 4),
                             minmax_GBps=round(N * bps / kernel_ms / 1e6, 1)))
    del f32, i8, qad

    ref = None
    try:
        import qt_fake
        from oracle import build_ref_path_creator

        mod = build_ref_path_creator.load()
        host = np.random.default_rng(2).standard_normal(1 << 26).astype(np.float32)
        spp = int(len(host) / 5000)
        with qt_fake.installed(mod):
            mod.create_path(host, 0, len(host))
            t0 = time.perf_counter()
            for _ in range(3):
                mod.create_path(host, 0, len(host))
            ms = (time.perf_counter() - t0) * 1e3 / 3
        ref = dict(samples=len(host), samples_per_pixel=spp, threads="1 (the reference parallelises only from 20000 samples per pixel)"
                   if spp < 20000 else "all", call_ms=round(ms, 2), cpu_count=os.cpu_count())
    except Exception as e:   # the reference is only there when oracle/_ref was built with its Python layer staged
        ref = dict(error="%s: %s" % (type(e).__name__, e))

    info = ctx.device_info()
    try:
        import subprocess

        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                               text=True).stdout.strip()
    except Exception:
        power = None
    result = dict(bench="view", gpu=info["name"], power_limit_and_max_sm_clock=power, log2n=args.log2n, reps=args.reps, rows=rows,
                  reference_create_path=ref)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
