"""Where the time of bench.py's step goes: one row per kernel of urh_demod_center_digitize on the bench capture.

    python tools/profile_step.py [--log2n 30] [--steps 5] [--warmup 3] [--timed 20] [--trace DIR]

The capture is built as bench.py builds it (urh_synth_fsk, same recipe and seeds).  After the warm-up the step runs --timed times
with the profiler off (CUDA events: the step's time) and then --steps times under torch.profiler with CUDA activities.  The trace is
cut into steps (every step launches the same kernels) and each row gives the median over the steps of a kernel's (or a memset's /
copy's) device time and of the idle gap before it.  The demodulation kernel is the longest one; the tail is the step's time minus
it.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the capture recipe and its constants)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def device_events(trace_path):
    """kernels, memsets and copies of the trace, in device order: (name, start_us, dur_us)"""
    with open(trace_path) as fh:
        tr = json.load(fh)
    ev = [(e["name"], float(e["ts"]), float(e["dur"])) for e in tr.get("traceEvents", [])
          if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    ev.sort(key=lambda e: e[1])
    return ev


def short(name, width=60):
    name = name.replace("(anonymous namespace)::", "")
    return name if len(name) <= width else name[: width - 3] + "..."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--steps", type=int, default=5, help="profiled steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--timed", type=int, default=20, help="steps timed with CUDA events, profiler off")
    ap.add_argument("--trace", metavar="DIR", help="keep the chrome trace in DIR (default: a temporary directory)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from urh_b200 import _lib
    from urh_b200.device import DeviceArray

    ctx = _lib.default_context(0)
    lib = ctx.lib
    torch.cuda.init()
    n = 1 << args.log2n
    nsym = n // bench.SPS + 2
    b, s = bench.make_symbols(nsym, seed=1000)
    d_b = DeviceArray(ctx, (nsym,), np.int8).set(b)
    d_s = DeviceArray(ctx, (nsym,), np.int32).set(s)
    d_iq = DeviceArray(ctx, (n, 2), np.float32)
    d_qad = DeviceArray(ctx, (n,), np.float32)
    ctx.check(lib.urh_synth_fsk(ctx.handle, C.c_void_p(d_iq.ptr), n, 0, bench.SPS, C.c_void_p(d_b.ptr), C.c_void_p(d_s.ptr),
                                C.c_double(bench.FDEV / bench.FS), 1.0, bench.SIGMA, 12345, 6_000_000, 5_000_000, *bench.capture_gaps(n, 0)))
    ctx.sync()

    rows = [0]

    def step():
        center, state, k = C.c_double(0.0), C.c_int(0), C.c_int64(0)
        ctx.check(lib.urh_demod_center_digitize(ctx.handle, C.c_void_p(d_iq.ptr), _lib.DT_F32, n, bench.NOISE_MAG, _lib.MOD_FSK, bench.TOL,
                                                bench.SPS, -1, C.c_void_p(d_qad.ptr), C.byref(center), C.byref(state), C.byref(k)))
        assert state.value == 1, "detect_center: state %d" % state.value
        rows[0] = k.value

    for _ in range(args.warmup):
        step()
    ctx.sync()
    launches0 = ctx.launch_count()
    ctx.timer_start()
    for _ in range(args.timed):
        step()
    ms_step = ctx.timer_stop() / args.timed
    launches = (ctx.launch_count() - launches0) // args.timed

    tdir = args.trace or tempfile.mkdtemp(prefix="profile_step_")
    os.makedirs(tdir, exist_ok=True)
    trace = os.path.join(tdir, "step.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        ctx.sync()
    prof.export_chrome_trace(trace)
    ev = device_events(trace)
    if len(ev) % args.steps:
        sys.exit("profile_step: %d device events do not split into %d equal steps" % (len(ev), args.steps))
    per = len(ev) // args.steps
    steps = [ev[i * per:(i + 1) * per] for i in range(args.steps)]
    names = [e[0] for e in steps[0]]
    if any([e[0] for e in st] != names for st in steps):
        sys.exit("profile_step: the profiled steps did not run the same kernels")
    dur = np.array([[e[2] for e in st] for st in steps]) / 1e3                                    # ms
    gap = np.array([[0.0] + [st[i][1] - (st[i - 1][1] + st[i - 1][2]) for i in range(1, per)] for st in steps]) / 1e3
    span = np.array([st[-1][1] + st[-1][2] - st[0][1] for st in steps]) / 1e3
    dmed, gmed = np.median(dur, axis=0), np.median(gap, axis=0)
    demod = int(np.argmax(dmed))

    print("card: %s" % card())
    print("capture: 2^%d float32 FSK samples (bench.py recipe), %d pulse rows; %d launches per step" % (args.log2n, rows[0], launches))
    print("%-3s %-60s %10s %10s" % ("#", "kernel / activity", "device ms", "gap ms"))
    for i in range(per):
        print("%-3d %-60s %10.4f %10.4f" % (i, short(names[i]), dmed[i], gmed[i]))
    after = slice(demod + 1, per)
    summary = {"card": card(), "log2n": args.log2n, "launches_per_step": launches, "ms_per_step": ms_step,
               "device_span_ms": float(np.median(span)), "demod_kernel": short(names[demod], 200), "demod_ms": float(dmed[demod]),
               "tail_ms": ms_step - float(dmed[demod]),
               "after_demod_busy_ms": float(dmed[after].sum()), "after_demod_gaps_ms": float(gmed[after].sum()),
               "kernels": [{"name": names[i], "ms": float(dmed[i]), "gap_ms": float(gmed[i])} for i in range(per)]}
    print("step (CUDA events, %d steps, profiler off): %.4f ms; demodulation kernel %.4f ms; tail %.4f ms "
          "(after the demodulation kernel: %.4f ms busy, %.4f ms idle gaps)"
          % (args.timed, ms_step, dmed[demod], summary["tail_ms"], summary["after_demod_busy_ms"], summary["after_demod_gaps_ms"]))
    print(json.dumps({k: v for k, v in summary.items() if k != "kernels"}))
    with open(os.path.join(tdir, "profile_step.json"), "w") as fh:
        json.dump(summary, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
