"""Streamed filters and dB map (the windowed ring, DESIGN.md §4.11) against the host-fed resident calls.

One process, pinned complex64 input and pinned outputs.  For each of band-pass (101 taps), FIR (10 taps), DC correction and the dB map
(W = 1024, hop 512) at each --log2n, the streamed C entry and the resident one fed from the host (upload, kernel, download, one after
the other) are alternated, --runs timed rounds after a warm-up round; the best time of each is reported.  Every line counts the 32-bit
words in which the two outputs differ (must be 0); the DC correction (double regime above 2^22 rows) is also counted against
x - float32(float64 mean).  The card's name and power limit are read in the same run.  --huge adds one band-pass over a capture larger
than the device (5 * 2^30 samples, 80 GiB pinned), checked against the resident call on windows around chunk edges; it reports
"not run" when the host cannot pin that much."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def fill(dst, seed=0):
    """a seeded complex64 pattern of 2^22 samples (a tone with random amplitude steps and noise), tiled over dst"""
    n0 = 1 << 22
    rng = np.random.default_rng(seed)
    t = np.arange(n0)
    x = (np.exp(2j * np.pi * 0.05 * t) * (1 + 0.5 * (rng.random(n0) > 0.5)) + 0.1 * (rng.standard_normal(n0) + 1j * rng.standard_normal(n0)))
    x = x.astype(np.complex64)
    for s in range(0, len(dst), n0):
        e = min(s + n0, len(dst))
        dst[s:e] = x[: e - s]


def words_differing(a, b, step=1 << 26):
    av, bv = a.reshape(-1).view(np.uint32), b.reshape(-1).view(np.uint32)
    return int(sum(np.count_nonzero(av[s: s + step] != bv[s: s + step]) for s in range(0, len(av), step)))


def dc_reference_differing(x, y, step=1 << 24):
    """words of y (float32 (n, 2)) that differ from x - float32(float64 mean)"""
    iq = x.view(np.float32).reshape(-1, 2)
    s = np.zeros(2, np.float64)
    for a in range(0, len(iq), step):
        s += iq[a: a + step].astype(np.float64).sum(axis=0)
    mean = (s / len(iq)).astype(np.float32)
    yv = y.view(np.float32).reshape(-1, 2)
    return int(sum(np.count_nonzero((iq[a: a + step] - mean).view(np.uint32) != yv[a: a + step].view(np.uint32))
                   for a in range(0, len(iq), step)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, nargs="+", default=[28, 30])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1 << 24)
    ap.add_argument("--ring", type=int, default=2)
    ap.add_argument("--entries", nargs="+", default=["bandpass", "fir", "dc", "db"])
    ap.add_argument("--huge", action="store_true")
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, PinnedArray
    from urh_b200.signalprocessing.Filter import Filter

    ctx = _lib.default_context()
    lib, h = ctx.lib, ctx.handle
    name = card()
    taps_bp = np.ascontiguousarray(Filter.bandpass_taps(-0.1, 0.2, 0.04), dtype=np.complex128)   # 101 taps
    taps_fir = np.ascontiguousarray(np.full(10, 0.1, np.complex64))
    W, hop = 1024, 512
    window = np.ascontiguousarray(np.hanning(W), dtype=np.float64)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    for log2n in args.log2n:
        n = 1 << log2n
        x = PinnedArray((n,), np.complex64)
        fill(x.array)
        d_x = DeviceArray(ctx, (n,), np.complex64)
        for entry in args.entries:
            m = len(taps_bp)
            frames = (n - W) // hop + 1
            out_shape, out_dtype = {"bandpass": ((n,), np.complex64), "fir": ((n,), np.complex64), "dc": ((n, 2), np.float32),
                                    "db": ((frames, W), np.float32)}[entry]
            outs = {k: PinnedArray(out_shape, out_dtype) for k in ("stream", "resident")}
            d_y = DeviceArray(ctx, out_shape, out_dtype)
            d_tb = DeviceArray(ctx, (m,), np.complex128).set(taps_bp)
            d_tf = DeviceArray(ctx, (10,), np.complex64).set(taps_fir)
            d_w = DeviceArray(ctx, (W,), np.float64).set(window)
            xp, ys, yr = C.c_void_p(x.ptr), C.c_void_p(outs["stream"].ptr), C.c_void_p(outs["resident"].ptr)

            def stream():
                if entry == "bandpass":
                    ctx.check(lib.urh_convolve_c128_stream(h, xp, n, P(taps_bp), m, (m - 1) // 2, n, args.chunk, args.ring, ys))
                elif entry == "fir":
                    ctx.check(lib.urh_fir_filter_stream(h, xp, n, P(taps_fir), 10, args.chunk, args.ring, ys))
                elif entry == "dc":
                    ctx.check(lib.urh_dc_correction_stream(h, xp, _lib.DT_F32, n, int(n <= Filter.EXACT_DC_MAX), args.chunk, args.ring, ys))
                else:
                    ctx.check(lib.urh_spectrogram_db_stream(h, xp, n, W, hop, P(window), frames, args.chunk, args.ring, ys))

            def resident():
                ctx.check(lib.urh_memcpy_h2d(h, C.c_void_p(d_x.ptr), xp, n * 8))
                dx, dy = C.c_void_p(d_x.ptr), C.c_void_p(d_y.ptr)
                if entry == "bandpass":
                    ctx.check(lib.urh_convolve_c128(h, dx, n, C.c_void_p(d_tb.ptr), m, (m - 1) // 2, n, dy))
                elif entry == "fir":
                    ctx.check(lib.urh_fir_filter(h, dx, n, C.c_void_p(d_tf.ptr), 10, dy))
                elif entry == "dc":
                    ctx.check(lib.urh_dc_correction(h, dx, n, dy, int(n <= Filter.EXACT_DC_MAX)))
                else:
                    ctx.check(lib.urh_spectrogram_db(h, dx, n, W, hop, C.c_void_p(d_w.ptr), frames, dy))
                ctx.check(lib.urh_memcpy_d2h(h, yr, C.c_void_p(d_y.ptr), d_y.nbytes))

            times = {"stream": [], "resident": []}
            for r in range(args.runs + 1):   # round 0 warms both up
                for kind, fn in (("stream", stream), ("resident", resident)):
                    ctx.sync()
                    t = time.perf_counter()
                    fn()
                    ctx.sync()
                    if r:
                        times[kind].append(time.perf_counter() - t)
            line = {"card": name, "entry": entry, "n": n, "chunk": args.chunk, "ring": args.ring,
                    "stream_s": [round(v, 4) for v in times["stream"]], "resident_s": [round(v, 4) for v in times["resident"]],
                    "stream_gsps": round(n / min(times["stream"]) / 1e9, 3), "resident_gsps": round(n / min(times["resident"]) / 1e9, 3),
                    "words_differing": words_differing(outs["stream"].array, outs["resident"].array)}
            line["stream_over_resident"] = round(min(times["resident"]) / min(times["stream"]), 3)
            if entry == "dc":
                line["words_differing_vs_f64_mean"] = dc_reference_differing(x.array, outs["stream"].array)
            print(json.dumps(line), flush=True)
            for o in outs.values():
                o.free()
            del d_y
        x.free()
        del d_x
    if args.huge:
        huge(ctx, args, name, taps_bp)


def huge(ctx, args, name, taps):
    """one band-pass over 5 * 2^30 complex64 samples (40 GiB in, 40 GiB out, pinned): more than the card holds"""
    from urh_b200.device import DeviceArray, PinnedArray

    n = 5 << 30
    m = len(taps)
    half = (m - 1) // 2
    try:
        x = PinnedArray((n,), np.complex64)
        y = PinnedArray((n,), np.complex64)
    except (MemoryError, RuntimeError) as e:
        print(json.dumps({"card": name, "entry": "bandpass", "n": n, "huge": "not run", "reason": str(e)[:200]}), flush=True)
        return
    fill(x.array, 1)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    ctx.sync()
    t = time.perf_counter()
    ctx.check(ctx.lib.urh_convolve_c128_stream(ctx.handle, C.c_void_p(x.ptr), n, P(taps), m, half, n, args.chunk, args.ring, C.c_void_p(y.ptr)))
    ctx.sync()
    dt = time.perf_counter() - t
    # the resident call on windows of 2^22 outputs around the first, middle and last chunk edges and the capture's ends
    L = 1 << 22
    edges = [0, args.chunk, (n // args.chunk // 2) * args.chunk, (n // args.chunk - 1) * args.chunk, n - L]
    d_t = DeviceArray(ctx, (m,), np.complex128).set(taps)
    diff = 0
    for e in edges:
        k0 = min(max(0, e - L // 2), n - L)
        a, b = max(0, k0 + half - (m - 1)), min(n, k0 + L + half)
        d_x = DeviceArray(ctx, (b - a,), np.complex64).set(x.array[a:b])
        d_y = DeviceArray(ctx, (L,), np.complex64)
        ctx.check(ctx.lib.urh_convolve_c128(ctx.handle, C.c_void_p(d_x.ptr), b - a, C.c_void_p(d_t.ptr), m, k0 + half - a, L, C.c_void_p(d_y.ptr)))
        diff += words_differing(d_y.get(), y.array[k0: k0 + L])
    print(json.dumps({"card": name, "entry": "bandpass", "n": n, "chunk": args.chunk, "ring": args.ring, "stream_s": round(dt, 3),
                      "stream_gsps": round(n / dt / 1e9, 3), "windows_checked": len(edges), "words_differing": diff}), flush=True)
    x.free()
    y.free()


if __name__ == "__main__":
    main()
