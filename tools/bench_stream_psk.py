"""Streamed PSK demodulation (urh_afp_demod_psk_stream) against the host-fed resident PSK call, in one process.

Pinned host captures of 2^log2n samples (float32 and int8) of PSK bursts with gaps.  The resident call uploads the capture, runs
urh_afp_demod(PSK) and downloads qad into pinned memory; the streamed call goes from the pinned capture to pinned qad through the
ring.  The two are alternated --runs times each after one warm-up round.  Prints one JSON line per (dtype, n, chunk): GS/s of each
call, the Costas loop alone on the device (resident, at n and at one chunk), the summed stitch counters of the streamed call,
whether qad agrees bit for bit, whether the rows of urh_demod_digitize_psk_stream equal urh_demod_digitize's, the first 2^22
samples against the CPU oracle, and the card's name and power limit read in the same run.  --big-log2n adds one streamed-only int8
run at a size the resident call cannot hold, when the host has the memory for it.

--trace SECONDS writes to stderr a timestamped line at every step of the bench, and every SECONDS the Python stack of every thread
(faulthandler), the GPU's utilisation and memory in use (nvidia-smi) and the host's load average: where a run spends its time, and
whether a slow step waits on the device or on the host."""
import argparse
import ctypes as C
import faulthandler
import json
import os
import subprocess
import sys
import threading
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


def fill(dst, dtype, order, seed=0):
    """PSK bursts (100 samples per symbol, carrier offset 0.01 cycles per sample) with gaps, 2^22 samples tiled over the capture"""
    n0 = 1 << 22
    rng = np.random.default_rng(seed)
    sym = rng.integers(0, order, n0 // 100 + 1)
    ph = 2 * np.pi * 0.01 * np.arange(n0) + np.repeat(2 * np.pi * sym / order, 100)[:n0]
    x = np.exp(1j * ph) + 0.05 * (rng.standard_normal(n0) + 1j * rng.standard_normal(n0))
    x[(np.arange(n0) % 60_000) > 50_000] *= 0.001
    iq = np.stack([x.real, x.imag], axis=1)
    iq = (iq * 100).astype(np.int8) if dtype == np.int8 else iq.astype(np.float32)
    for s in range(0, len(dst), n0):
        e = min(s + n0, len(dst))
        dst[s:e] = iq[: e - s]


NOISE = {np.float32: 0.2, np.int8: 20.0}


def host_free_bytes():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


T0 = time.perf_counter()
TRACE = False


def step(what, **kw):
    """one timestamped progress line on stderr (--trace)"""
    if TRACE:
        print(json.dumps({"t": round(time.perf_counter() - T0, 2), "step": what, **kw}), file=sys.stderr, flush=True)


def watch(period):
    """every `period` seconds: the Python stacks, the GPU's utilisation and memory in use, the host's load average (stderr)"""
    faulthandler.dump_traceback_later(period, repeat=True, file=sys.stderr)

    def loop():
        while True:
            time.sleep(period)
            try:
                gpu = subprocess.run(["nvidia-smi", "--query-gpu=utilization.gpu,memory.used,clocks.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
            except (OSError, subprocess.SubprocessError):
                gpu = "unknown"
            try:
                with open("/proc/loadavg") as f:
                    load = f.read().strip()
            except OSError:
                load = "unknown"
            step("watch", gpu=gpu, load=load)

    threading.Thread(target=loop, daemon=True).start()


def costas_stats(ctx):
    st3, st4 = (C.c_int64 * 3)(), (C.c_int64 * 4)()
    ctx.check(ctx.lib.urh_costas_stats(ctx.handle, st3))
    ctx.check(ctx.lib.urh_costas_stitch_stats(ctx.handle, st4))
    return dict(zip(("fast", "walked", "stepped", "A", "B", "self", "segs"), list(st3) + list(st4)))


def device_ms(ctx, lib_call, reps=3):
    """best wall time of a device-only call between two synchronisations"""
    best = None
    for _ in range(reps + 1):
        ctx.sync()
        t = time.perf_counter()
        lib_call()
        ctx.sync()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, nargs="+", default=[28, 30])
    ap.add_argument("--order", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--dtype", nargs="+", default=["float32", "int8"])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--chunk", type=int, nargs="+", default=None, help="ring chunk samples (default: PSK_STREAM_CHUNK)")
    ap.add_argument("--ring", type=int, default=2)
    ap.add_argument("--big-log2n", type=int, default=0)
    ap.add_argument("--no-digitize", action="store_true")
    ap.add_argument("--trace", type=float, default=0, help="progress lines and a stack / GPU / load sample every TRACE seconds")
    args = ap.parse_args()
    global TRACE
    if args.trace > 0:
        TRACE = True
        watch(args.trace)
    from oracle import oracle
    from urh_b200 import _lib
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import DeviceArray, PinnedArray

    oracle.build()
    ctx = _lib.default_context()
    name = card()
    chunks = args.chunk or [sf.PSK_STREAM_CHUNK]
    for log2n in args.log2n:
        n = 1 << log2n
        for dname in args.dtype:
            dtype = np.dtype(dname).type
            noise = NOISE[dtype]
            code = _lib.dtype_code(dtype)
            for order in args.order:
                cfg = {"dtype": dname, "n": n, "order": order}
                step("pinned alloc", **cfg)
                host = PinnedArray((n, 2), dtype)
                step("fill", **cfg)
                fill(host.array, dtype, order)
                q_host = {kind: PinnedArray((n,), np.float32) for kind in ("stream", "resident")}
                step("device alloc", **cfg)
                d_iq = DeviceArray(ctx, (n, 2), dtype)
                d_qad = DeviceArray(ctx, (n,), np.float32)

                def resident():
                    ctx.check(ctx.lib.urh_memcpy_h2d(ctx.handle, C.c_void_p(d_iq.ptr), C.c_void_p(host.ptr), n * 2 * np.dtype(dtype).itemsize))
                    ctx.check(ctx.lib.urh_afp_demod(ctx.handle, C.c_void_p(d_iq.ptr), code, n, noise, _lib.MOD_PSK, order, 0.1,
                                                    C.c_void_p(d_qad.ptr)))
                    d_qad.get(out=q_host["resident"].array)

                # the Costas loop alone on the device, over the whole capture and over one chunk's worth of it
                step("upload", **cfg)
                d_iq.set_async(host.array)
                step("device-only loop", **cfg)
                dev_full = device_ms(ctx, lambda: ctx.check(ctx.lib.urh_afp_demod(ctx.handle, C.c_void_p(d_iq.ptr), code, n, noise, _lib.MOD_PSK,
                                                                                   order, 0.1, C.c_void_p(d_qad.ptr))))
                for cs in chunks:
                    def stream():
                        ctx.check(ctx.lib.urh_afp_demod_psk_stream(ctx.handle, C.c_void_p(host.ptr), code, n, noise, order, 0.1, cs, args.ring,
                                                                   C.c_void_p(q_host["stream"].ptr)))

                    m = min(cs, n)
                    dev_chunk = device_ms(ctx, lambda: ctx.check(ctx.lib.urh_afp_demod(ctx.handle, C.c_void_p(d_iq.ptr), code, m, noise,
                                                                                        _lib.MOD_PSK, order, 0.1, C.c_void_p(d_qad.ptr))))
                    res = {"stream": [], "resident": []}
                    for r in range(args.runs + 1):
                        for kind, call in (("stream", stream), ("resident", resident)):
                            ctx.sync()
                            step(kind, run=r, chunk=cs, **cfg)
                            t = time.perf_counter()
                            call()
                            ctx.sync()
                            dt = time.perf_counter() - t
                            if kind == "stream" and r == args.runs:
                                st = costas_stats(ctx)
                            if r > 0:
                                res[kind].append(dt)
                    qs, qr = q_host["stream"].array, q_host["resident"].array
                    nan_s, nan_r = np.isnan(qs), np.isnan(qr)
                    identical = bool(np.array_equal(nan_s, nan_r) and (qs.view(np.uint32)[~nan_r] == qr.view(np.uint32)[~nan_r]).all())
                    w = min(n, 1 << 22)
                    step("oracle", **cfg)
                    ref = oracle.afp_demod(np.ascontiguousarray(host.array[:w]), noise, "PSK", order, 0.1)
                    oracle_diff = int(np.count_nonzero(qs[1:w].view(np.uint32) != ref[1:w].view(np.uint32)))
                    rows_same = None
                    if not args.no_digitize and order in (2, 4):
                        bps = 1 if order == 2 else 2
                        k0, k1 = C.c_int64(0), C.c_int64(0)
                        step("resident demod_digitize", **cfg)
                        ctx.check(ctx.lib.urh_demod_digitize(ctx.handle, C.c_void_p(d_iq.ptr), code, n, noise, _lib.MOD_PSK, 0.0, 5, 100, bps, 0.5,
                                                             C.c_void_p(d_qad.ptr), C.byref(k0)))
                        r0 = sf._fetch_pulses(ctx, k0.value).copy()
                        step("streamed demod_digitize", rows=len(r0), **cfg)
                        ctx.check(ctx.lib.urh_demod_digitize_psk_stream(ctx.handle, C.c_void_p(host.ptr), code, n, noise, 0.0, 5, 100, bps, 0.5,
                                                                        cs, args.ring, C.c_void_p(q_host["stream"].ptr), C.byref(k1)))
                        r1 = sf._fetch_pulses(ctx, k1.value)
                        step("compare", **cfg)
                        rows_same = bool(np.array_equal(r0, r1)) and bool(
                            (d_qad.get().view(np.uint32) == q_host["stream"].array.view(np.uint32)).all())
                    print(json.dumps({
                        "card": name, "dtype": dname, "n": n, "order": order, "chunk": cs, "ring": args.ring,
                        "stream_s": [round(x, 4) for x in res["stream"]], "resident_s": [round(x, 4) for x in res["resident"]],
                        "stream_gsps": round(n / min(res["stream"]) / 1e9, 3), "resident_gsps": round(n / min(res["resident"]) / 1e9, 3),
                        "costas_device_gsps": round(n / dev_full / 1e9, 3), "costas_device_one_chunk_gsps": round(m / dev_chunk / 1e9, 3),
                        "stream_costas_stats": st, "qad_identical": identical, "dd_rows_and_qad_identical": rows_same,
                        "oracle_first_2p22_words_differing": oracle_diff,
                    }), flush=True)
                step("free", **cfg)
                qs = qr = nan_s = nan_r = None   # views of the pinned buffers freed below
                del d_iq, d_qad
                for a in q_host.values():
                    a.free()
                host.free()
    if args.big_log2n:
        n = 1 << args.big_log2n
        need = n * 2 + n * 4
        if host_free_bytes() < need + (8 << 30):
            print(json.dumps({"card": name, "dtype": "int8", "n": n, "streamed_only": "not measured: host memory",
                              "host_available": host_free_bytes(), "needed": need}), flush=True)
            return
        step("pinned alloc", dtype="int8", n=n)
        host = PinnedArray((n, 2), np.int8)
        step("fill", dtype="int8", n=n)
        fill(host.array, np.int8, 4)
        q = PinnedArray((n,), np.float32)
        step("stream", dtype="int8", n=n)
        ctx.sync()
        t = time.perf_counter()
        ctx.check(ctx.lib.urh_afp_demod_psk_stream(ctx.handle, C.c_void_p(host.ptr), _lib.DT_I8, n, NOISE[np.int8], 4, 0.1, chunks[0], args.ring,
                                                   C.c_void_p(q.ptr)))
        ctx.sync()
        dt = time.perf_counter() - t
        w = 1 << 22
        ref = oracle.afp_demod(np.ascontiguousarray(host.array[:w]), NOISE[np.int8], "PSK", 4, 0.1)
        resident_bytes = sf.stream_footprint(n, np.int8, 0, _lib.STREAM_AFP_DEMOD | sf.psk_entry(4) | _lib.STREAM_RESIDENT, rows=-2)
        print(json.dumps({"card": name, "dtype": "int8", "n": n, "order": 4, "chunk": chunks[0], "streamed_only": True,
                          "stream_s": round(dt, 3), "stream_gsps": round(n / dt / 1e9, 3), "resident_footprint_bytes": resident_bytes,
                          "stream_costas_stats": costas_stats(ctx),
                          "oracle_first_2p22_words_differing": int(np.count_nonzero(q.array[1:w].view(np.uint32) != ref[1:w].view(np.uint32)))}),
              flush=True)
        q.free()
        host.free()


if __name__ == "__main__":
    main()
