#!/usr/bin/env python
"""Spectrogram STFT -> dB (W = 1024, hop 512): the fused shared-memory-FFT kernel against the cuFFT path (URH_B200_STFT_CUFFT=1),
and their agreement; create_image_segments, fused image kernel against the composed dB map + look-up; FTA record generation and
export.   python tools/bench_stft.py [--log2n 28]"""
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
    W, hop = 1024, 512
    frames = (n - W) // hop + 1
    d_w = to_device(np.hanning(W), ctx)
    out = {}
    res = {}
    for name, env in (("fused", None), ("cufft", "1")):
        if env:
            os.environ["URH_B200_STFT_CUFFT"] = env
        else:
            os.environ.pop("URH_B200_STFT_CUFFT", None)
        d_db = DeviceArray(ctx, (frames, W), np.float32)
        ms = []
        for rep in range(args.reps + 1):
            ctx.timer_start()
            ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr), frames, C.c_void_p(d_db.ptr)))
            t = ctx.timer_stop()
            if rep:
                ms.append(t)
        out[name + "_ms"] = float(np.median(ms))
        res[name] = d_db[:4096].get()
        d_db.free()
    peak = res["cufft"].max()
    mask = res["cufft"] > peak - 100
    out["max_abs_dB_diff_within_100dB_of_peak"] = float(np.abs(res["fused"] - res["cufft"])[mask].max())
    out["samples"] = n
    out["algorithmic_GBps_fused"] = 16.0 * n / out["fused_ms"] / 1e6
    os.environ.pop("URH_B200_STFT_CUFFT", None)
    out.update(bench_images(ctx, d_x, n, W, hop, d_w, args.reps))
    out.update(bench_fta(ctx, args.reps))
    info = ctx.device_info()
    out["device"] = info["name"]
    out["power_limit_W"] = power_limit()
    print(json.dumps(out))


def power_limit():
    """the enforced power limit, read (not set) through nvidia-smi; None where it cannot be read"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def bench_images(ctx, d_x, n, W, hop, d_w, reps):
    """create_image_segments at n samples: the fused image kernel (one launch for every segment) against the composed stages
    (urh_spectrogram_db then urh_bgra_lookup, per segment, as the reference's generator calls them), CUDA events"""
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    lib = ctx.lib
    spec = Spectrogram(d_x, W, 0.5)
    bounds = spec.segment_bounds()
    cmap = np.zeros((256, 4), np.uint8)
    cmap[:, 0] = np.arange(256)
    d_map = to_device(cmap, ctx)
    starts = np.array([s for s, _, _ in bounds], np.int64)
    lens = np.array([e - s for s, e, _ in bounds], np.int64)
    pixels = sum(f for _, _, f in bounds) * W
    d_img = DeviceArray(ctx, (pixels * 4,), np.uint8)
    max_f = max(f for _, _, f in bounds)
    d_db = DeviceArray(ctx, (max_f, W), np.float32)
    res = {"fused": [], "composed": []}
    for rep in range(reps + 1):
        ctx.timer_start()
        ctx.check(lib.urh_spectrogram_bgra(ctx.handle, C.c_void_p(d_x.ptr), n, W, hop, C.c_void_p(d_w.ptr), starts.ctypes.data_as(C.c_void_p),
                                           lens.ctypes.data_as(C.c_void_p), len(bounds), C.c_void_p(d_map.ptr), 256, -140.0, 10.0, 0,
                                           C.c_void_p(d_img.ptr)))
        t_fused = ctx.timer_stop()
        ctx.timer_start()
        off = 0
        for s, e, f in bounds:
            ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr + 8 * s), e - s, W, hop, C.c_void_p(d_w.ptr), f, C.c_void_p(d_db.ptr)))
            ctx.check(lib.urh_bgra_lookup(ctx.handle, C.c_void_p(d_db.ptr), f, W, C.c_void_p(d_map.ptr), 256, -140.0, 10.0, 1,
                                          C.c_void_p(d_img.ptr + off)))
            off += f * W * 4
        t_comp = ctx.timer_stop()
        if rep:
            res["fused"].append(t_fused)
            res["composed"].append(t_comp)
    out = {"image_segments": len(bounds), "image_fused_ms": float(np.median(res["fused"])),
           "image_composed_ms": float(np.median(res["composed"]))}
    out["image_fused_GBps_8B_per_sample"] = 8.0 * n / out["image_fused_ms"] / 1e6
    return out


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
