#!/usr/bin/env python
"""Spectrogram at 2^log2n samples, hop W/2, for each window size W: the dB map (urh_spectrogram_db) and the images of every
create_image_segments segment in one call (urh_spectrogram_bgra), CUDA events; FTA record generation and export.
   python tools/bench_stft.py [--log2n 28] [--windows 128 256 512 1024 2048 4096]"""
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
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--windows", type=int, nargs="+", default=[128, 256, 512, 1024, 2048, 4096])
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device

    ctx = _lib.default_context()
    lib = ctx.lib
    n = 1 << args.log2n
    rng = np.random.default_rng(0)
    chunk = (rng.standard_normal((1 << 20, 2)) * 0.1).astype(np.float32)
    chunk[:, 0] += np.cos(2 * np.pi * 0.05 * np.arange(1 << 20)).astype(np.float32)
    chunk[:, 1] += np.sin(2 * np.pi * 0.05 * np.arange(1 << 20)).astype(np.float32)
    d_x = DeviceArray(ctx, (n, 2), np.float32)
    d_c = to_device(chunk, ctx)
    for i in range(n >> 20):
        ctx.check(lib.urh_memcpy_d2d(ctx.handle, C.c_void_p(d_x.ptr + i * chunk.nbytes), C.c_void_p(d_c.ptr), chunk.nbytes))
    out = {"samples": n}
    for W in args.windows:
        out.update(bench_window(ctx, d_x, n, W, args.reps))
    out.update(bench_fta(ctx, args.reps))
    info = ctx.device_info()
    out["device"] = info["name"]
    out["power_limit_W"] = power_limit()
    print(json.dumps(out))


def timed(ctx, reps, call):
    """median over reps calls, after one warm-up call, of the CUDA-event time of call()"""
    ms = []
    for rep in range(reps + 1):
        ctx.timer_start()
        call()
        t = ctx.timer_stop()
        if rep:
            ms.append(t)
    return float(np.median(ms))


def power_limit():
    """the enforced power limit, read (not set) through nvidia-smi; None where it cannot be read"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def bench_window(ctx, d_x, n, W, reps):
    """at window size W, hop W/2: the dB map of every frame, and the images of create_image_segments' segments in one call (256
    colormap entries, (min, max) = (-140, 10), the scene view's layout)"""
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    lib = ctx.lib
    hop = W // 2
    frames = (n - W) // hop + 1
    d_w = to_device(np.hanning(W), ctx)
    d_db = DeviceArray(ctx, (frames, W), np.float32)
    db_ms = timed(ctx, reps, lambda: ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr),
                                                                      frames, C.c_void_p(d_db.ptr))))
    d_db.free()
    bounds = Spectrogram.segment_bounds_of(n, W, hop)
    cmap = np.zeros((256, 4), np.uint8)
    cmap[:, 0] = np.arange(256)
    d_map = to_device(cmap, ctx)
    starts = np.array([s for s, _, _ in bounds], np.int64)
    lens = np.array([e - s for s, e, _ in bounds], np.int64)
    d_img = DeviceArray(ctx, (sum(f for _, _, f in bounds) * W * 4,), np.uint8)
    image_ms = timed(ctx, reps, lambda: ctx.check(lib.urh_spectrogram_bgra(
        ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr), starts.ctypes.data_as(C.c_void_p),
        lens.ctypes.data_as(C.c_void_p), len(bounds), C.c_void_p(d_map.ptr), 256, -140.0, 10.0, 0, C.c_void_p(d_img.ptr))))
    d_img.free()
    k = "W%d_" % W
    return {k + "db_ms": db_ms, k + "db_GBps_16B_per_sample": 16.0 * n / db_ms / 1e6, k + "image_segments": len(bounds),
            k + "image_ms": image_ms, k + "image_GBps_8B_per_sample": 8.0 * n / image_ms / 1e6}


def bench_fta(ctx, reps, log2n=23, sample_rate=2e6):
    """FTA records at 2^log2n samples (W = 1024): generation on the device in GB/s (48 B per cell, no disk), and the wall time of
    export_to_fta including the file write (to a temporary directory)"""
    import tempfile
    import time
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    lib = ctx.lib
    n, W = 1 << log2n, 1024
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    spec = Spectrogram(x, W, 0.5)
    d_db = spec._run(x, 1, keep=True)
    F = d_db.shape[0]
    freqs = to_device(np.fft.fftshift(np.fft.fftfreq(W, 1 / sample_rate)), ctx)
    tw = 1e9 * ((n / sample_rate) / F)
    d_out = DeviceArray(ctx, (W * F * 48,), np.uint8)
    ms = []
    for rep in range(reps + 1):
        ctx.timer_start()
        ctx.check(lib.urh_fta_records(ctx.handle, C.c_void_p(d_db.ptr), F, W, 0, W, C.c_void_p(freqs.ptr), tw, 1, C.c_void_p(d_out.ptr), None))
        t = ctx.timer_stop()
        if rep:
            ms.append(t)
    d_out.free()
    out = {"fta_samples": n, "fta_bytes": W * F * 48, "fta_records_ms": float(np.median(ms))}
    out["fta_records_GBps"] = W * F * 48 / out["fta_records_ms"] / 1e6
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        spec.export_to_fta(sample_rate, os.path.join(tmp, "x.fta"), True)
        out["fta_export_wall_s"] = time.perf_counter() - t0
    return out


if __name__ == "__main__":
    main()
