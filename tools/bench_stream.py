"""Streamed one-call step (urh_demod_center_digitize_stream) against the host-fed resident step (urh_demod_center_digitize_host).

One process, pinned host captures of 2^log2n samples (float32 and int8), the two calls alternated --runs times each.  Prints one
JSON line per dtype: GS/s and H2D GB/s of each call, whether center, rows and qad agree bit for bit, and the card's name and power
limit read in the same run.  The streamed result is also checked against the CPU oracle (the reference's compiled kernels when
oracle/_ref travelled, else the C restatement), as bench.py does, on windows of 2^22 samples that straddle the first, middle and
last chunk edges plus the capture's first and last samples: every qad word and every pulse boundary inside a window."""
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


def fill(dst, dtype, seed=0):
    """a 2-FSK burst pattern of 2^22 samples, tiled over the capture"""
    n0 = 1 << 22
    rng = np.random.default_rng(seed)
    f = np.repeat(np.where(rng.integers(0, 2, n0 // 100 + 1) > 0, 0.01, -0.01), 100)[:n0]
    x = np.exp(2j * np.pi * np.cumsum(f)) + 0.01 * (rng.standard_normal(n0) + 1j * rng.standard_normal(n0))
    x[(np.arange(n0) % 60_000) > 50_000] *= 0.001
    iq = np.stack([x.real, x.imag], axis=1)
    iq = (iq * 100).astype(np.int8) if dtype == np.int8 else iq.astype(np.float32)
    for s in range(0, len(dst), n0):
        e = min(s + n0, len(dst))
        dst[s:e] = iq[: e - s]


TOL, SPS = 5, 100


def oracle_kernels():
    from oracle import oracle, ref_loader

    try:
        sfr, _, _ = ref_loader.load_kernels()
        return (lambda iq, nm: np.asarray(sfr.afp_demod(iq, nm, "FSK", 2)),
                lambda q, c: np.asarray(sfr.grab_pulse_lens(q, c, TOL, "FSK", SPS)), "reference")
    except Exception:
        oracle.build()
        return (lambda iq, nm: np.asarray(oracle.afp_demod(iq, nm, "FSK", 2)),
                lambda q, c: np.asarray(oracle.grab_pulse_lens(q, c, TOL, "FSK", SPS)), "port")


def parity(host_iq, noise, d_qad, rows, center, n, chunk, w=1 << 22):
    """bench.py's parity block for one GPU, with windows placed across chunk edges"""
    demod, grab, kind = oracle_kernels()
    edges = list(range(chunk, n, chunk))
    centers = sorted({0, n} | ({edges[0], edges[len(edges) // 2], edges[-1]} if edges else set()))
    starts = sorted({min(max(0, c - w // 2), n - w) for c in centers}) if n > w else [0]
    w = min(w, n)
    pos_gpu = TOL - 1 + np.cumsum(rows[:-1, 1])
    st_gpu = rows[:-1, 0]
    margin = min(w // 4, 1 << 20)
    out = {"oracle": kind, "window_samples": w, "windows": len(starts), "qad_words_differing": 0, "boundaries_compared": 0,
           "boundaries_differing": 0}
    for a in starts:
        iq = np.ascontiguousarray(host_iq[max(a - 1, 0): a + w])
        q_ref = demod(iq, noise)
        if a > 0:
            q_ref = q_ref[1:]
        q_gpu = d_qad[a: a + w].get()
        out["qad_words_differing"] += int(np.count_nonzero(q_gpu.view(np.uint32) != q_ref.view(np.uint32)))
        r_ref = grab(np.ascontiguousarray(q_ref), float(center))
        pos_ref = a + TOL - 1 + np.cumsum(r_ref[:-1, 1])
        st_ref = r_ref[:-1, 0]
        lo, hi = a + (margin if a > 0 else -1), a + w
        mg = (pos_gpu > lo) & (pos_gpu < hi)
        mr = (pos_ref > lo) & (pos_ref < hi)
        pg, sg, pr, sr = pos_gpu[mg], st_gpu[mg], pos_ref[mr], st_ref[mr]
        out["boundaries_compared"] += int(len(pr))
        if len(pg) != len(pr):
            out["boundaries_differing"] += abs(len(pg) - len(pr)) + 1
        else:
            out["boundaries_differing"] += int(np.count_nonzero((pg != pr) | (sg != sr)))
    out["ok"] = out["qad_words_differing"] == 0 and out["boundaries_differing"] == 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1 << 24)
    ap.add_argument("--ring", type=int, default=2)
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.cythonext.signal_functions import _fetch_pulses
    from urh_b200.device import DeviceArray, PinnedArray

    ctx = _lib.default_context()
    n = 1 << args.log2n
    name = card()
    for dtype, noise in ((np.float32, 0.05), (np.int8, 5.0)):
        host = PinnedArray((n, 2), dtype)
        fill(host.array, dtype)
        ptr = C.c_void_p(host.ptr)
        code = _lib.dtype_code(dtype)
        # separate qad buffers, NaN-filled: a sample one call fails to write cannot match the other's
        d_qad = {kind: DeviceArray(ctx, (n,), np.float32) for kind in ("stream", "host")}
        for d in d_qad.values():
            ctx.check(ctx.lib.urh_memset(ctx.handle, C.c_void_p(d.ptr), 0xFF, 4 * n))
        res = {"stream": [], "host": []}
        out = {}
        scratch = DeviceArray(ctx, (n, 2), dtype)
        for r in range(args.runs + 1):   # the first round warms both up
            for kind in ("stream", "host"):
                c, st, k, kept = C.c_double(0), C.c_int(0), C.c_int64(0), C.c_int64(0)
                ctx.sync()
                t = time.perf_counter()
                if kind == "stream":
                    ctx.check(ctx.lib.urh_demod_center_digitize_stream(ctx.handle, ptr, code, n, noise, _lib.MOD_FSK, 5, 100, -1, args.chunk,
                                                                       args.ring, C.c_void_p(d_qad["stream"].ptr), None, C.byref(c), C.byref(st),
                                                                       C.byref(kept), C.byref(k)))
                else:
                    ctx.check(ctx.lib.urh_demod_center_digitize_host(ctx.handle, ptr, code, n, noise, _lib.MOD_FSK, 5, 100, -1, args.chunk,
                                                                     C.c_void_p(scratch.ptr), C.c_void_p(d_qad["host"].ptr), C.byref(c), C.byref(st),
                                                                     C.byref(k)))
                ctx.sync()
                dt = time.perf_counter() - t
                if r > 0:
                    res[kind].append(dt)
                if r == args.runs:
                    out[kind] = (c.value, st.value, _fetch_pulses(ctx, k.value).copy(), d_qad[kind].get())
        same = (out["stream"][0] == out["host"][0] and out["stream"][1] == out["host"][1]
                and np.array_equal(out["stream"][2], out["host"][2])
                and bool((out["stream"][3].view(np.uint32) == out["host"][3].view(np.uint32)).all()))
        del scratch
        par = parity(host.array, noise, d_qad["stream"], out["stream"][2], out["stream"][0], n, args.chunk)
        b = n * 2 * np.dtype(dtype).itemsize
        print(json.dumps({
            "card": name, "dtype": np.dtype(dtype).name, "n": n, "chunk": args.chunk, "ring": args.ring,
            "stream_s": [round(x, 4) for x in res["stream"]], "host_s": [round(x, 4) for x in res["host"]],
            "stream_gsps": round(n / min(res["stream"]) / 1e9, 3), "host_gsps": round(n / min(res["host"]) / 1e9, 3),
            "stream_h2d_gbps": round(b / min(res["stream"]) / 1e9, 2), "host_h2d_gbps": round(b / min(res["host"]) / 1e9, 2),
            "rows": len(out["host"][2]), "identical": same, "parity": par,
        }), flush=True)
        del d_qad
        host.free()


if __name__ == "__main__":
    main()
