"""Time IQArray.export_to_sub's device body (urh_sub_export) on captures resident in HBM, and the reference's export on a host slice.

    python tools/bench_sub_export.py [--log2n 30] [--reps 10] [--stream-log2n 28] [--ref-log2n 20] [--out FILE]

Captures are generated on the device (torch) from a seed: "ook" is runs of 0 and 255 with lengths uniform in 1 .. 6000 (1 % of them a
single sample, 1 % another value), "noise" is uniform over all 256 values (mostly one-sample runs and skips of ~256 samples).  Each
is timed as float32 and int8 with CUDA events around the whole call (it ends in a synchronise: the body's length is read back),
after one warm-up call.  The streamed export (urh_sub_export_stream) of a host float32 OOK-like capture of 2^stream-log2n samples in
pageable memory is timed with the host clock, file write to a temporary directory included, chunks of 2^24 samples, a ring of 2.
Bytes counted: the capture once plus the body written.  GS/s is samples over time; the share of HBM peak
is those bytes over time over 3.35 TB/s (H100 SXM data sheet).  The reference's export_to_sub (its Python loop, oracle/_ref when
built) is timed on a 2^ref-log2n-sample host slice on one core.  Prints one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12


def make_column(torch, kind, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "noise":
        return torch.randint(0, 256, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    runs = n // 3000 + 16
    lengths = torch.randint(1, 6001, (runs,), generator=g, device="cuda")
    lengths[torch.rand(runs, generator=g, device="cuda") < 0.01] = 1
    vals = (torch.arange(runs, device="cuda") % 2) * 255
    other = torch.rand(runs, generator=g, device="cuda") < 0.01
    vals[other] = torch.randint(0, 256, (runs,), generator=g, device="cuda")[other]
    col = torch.repeat_interleave(vals.to(torch.uint8), lengths)
    while col.numel() < n:
        col = torch.cat([col, col])
    return col[:n].contiguous()


def as_capture(torch, col, dtype):
    """an (n, 2) capture whose convert_to(uint8)[:, 0] is col"""
    if dtype == "int8":
        i = (col.to(torch.int16) - 128).to(torch.int8)
    else:
        i = (col.to(torch.float32) + 0.5) / 127 - 1
    return torch.stack([i, torch.zeros_like(i)], dim=1).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--stream-log2n", type=int, default=28)
    ap.add_argument("--ref-log2n", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from urh_b200 import _lib
    from urh_b200.device import DeviceArray

    ctx = _lib.default_context()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    n = 1 << args.log2n
    cap = int(ctx.lib.urh_sub_export_bound(n))
    body = DeviceArray(ctx, (cap,), np.uint8)
    result = {"n": n, "gpu": torch.cuda.get_device_name(0), "resident": {}}
    for kind in ("ook", "noise"):
        col = make_column(torch, kind, n, 1)
        for dtype in ("float32", "int8"):
            x = as_capture(torch, col, dtype)
            torch.cuda.synchronize()
            code = _lib.DT_F32 if dtype == "float32" else _lib.DT_I8
            nbytes = C.c_int64(0)

            def call():
                ctx.check(ctx.lib.urh_sub_export(ctx.handle, C.c_void_p(x.data_ptr()), code, n, C.c_void_p(body.ptr), cap,
                                                 C.byref(nbytes)))

            call()
            times = []
            for _ in range(args.reps):
                ctx.timer_start()
                call()
                times.append(ctx.timer_stop())
            ms = float(np.median(times))
            moved = x.numel() * x.element_size() + nbytes.value
            result["resident"]["%s_%s" % (kind, dtype)] = {
                "ms_median": round(ms, 3), "ms_min": round(min(times), 3), "body_bytes": nbytes.value,
                "gsps": round(n / ms / 1e6, 2), "hbm_fraction": round(moved / (ms * 1e-3) / HBM_PEAK, 3)}
            del x
        del col
        torch.cuda.empty_cache()
    body.free()

    m = 1 << args.stream_log2n
    host = as_capture(torch, make_column(torch, "ook", m, 2), "float32").cpu().numpy()
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        times = []
        for _ in range(3):
            fd = os.open(os.path.join(d, "s.sub"), os.O_WRONLY | os.O_CREAT | os.O_TRUNC)
            nbytes = C.c_int64(0)
            t = time.perf_counter()
            ctx.check(ctx.lib.urh_sub_export_stream(ctx.handle, host.ctypes.data_as(C.c_void_p), _lib.DT_F32, m, fd, 1 << 24, 2,
                                                    C.byref(nbytes)))
            times.append(time.perf_counter() - t)
            os.close(fd)
    s = float(np.median(times))
    result["streamed_host_float32"] = {"n": m, "s_median": round(s, 4), "body_bytes": nbytes.value, "gsps": round(m / s / 1e9, 2),
                                       "host_read_gbps": round(host.nbytes / s / 1e9, 2)}
    del host

    # the reference's loop on a host slice, for scale
    try:
        from oracle import ref_loader
        ref = ref_loader.load_python_layer()
        m = 1 << args.ref_log2n
        col = np.random.default_rng(1).integers(0, 256, m).astype(np.uint8)
        data = np.stack([col, col], axis=1)
        with tempfile.TemporaryDirectory() as d:
            t = time.perf_counter()
            ref.IQArray(data).export_to_sub(os.path.join(d, "r.sub"))
            s = time.perf_counter() - t
        result["reference_host"] = {"n": m, "s": round(s, 3), "msps": round(m / s / 1e6, 3)}
    except ImportError as e:
        result["reference_host"] = "not measured (%s)" % e
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
