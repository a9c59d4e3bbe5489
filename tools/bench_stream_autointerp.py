"""Streamed auto-interpretation (noise level, message segmentation, estimate(), DESIGN.md §4.11) against the resident path.

One process, pinned captures of 2^--log2n samples, float32 and int8: FSK bursts of 100 bits at 50 samples per bit between quiet gaps, a
seeded 2^22-sample pattern tiled over the capture, its last 5 % quiet.  For each dtype, detect_noise_level_iq, segment_messages_iq, estimate() and the chain
Signal -> auto_detect -> get_protocol_from_signal are timed streamed (the device budget forced to 1 MiB, so every step takes its host path)
and resident (no forced budget), alternated, best of --runs after a warm-up round.  Each line records whether the streamed result equals
the resident one.  The card's name and power limit are read in the same run.  --huge adds one streamed estimate() over a capture larger
than the device when the host can pin it, and reports "not run" otherwise."""
import argparse
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
    """FSK bursts between quiet gaps, a 2^22-sample pattern tiled over dst ((n, 2) float32 or int8)"""
    n0 = 1 << 22
    rng = np.random.default_rng(seed)
    x = np.zeros(n0, np.complex128)
    period = n0 // 16
    for k in range(16):
        bits = np.repeat(rng.integers(0, 2, 100), 50)
        s = k * period + 20_000
        x[s:s + len(bits)] = 0.8 * np.exp(1j * np.cumsum(np.where(bits > 0, 0.3, -0.3)))
    x += 0.01 * (rng.standard_normal(n0) + 1j * rng.standard_normal(n0))
    iq = np.stack([x.real, x.imag], 1)
    iq = iq.astype(np.float32) if dst.dtype == np.float32 else np.clip(np.rint(iq * 127), -128, 127).astype(np.int8)
    for s in range(0, len(dst), n0):
        e = min(s + n0, len(dst))
        dst[s:e] = iq[: e - s]
    # the last 5 % carry no bursts: the noise level has quiet chunks to find
    quiet = iq[:20_000]
    for s in range(len(dst) - len(dst) // 20, len(dst), len(quiet)):
        e = min(s + len(quiet), len(dst))
        dst[s:e] = quiet[: e - s]


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def steps(iq):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.ProtocolAnalyzer import ProtocolAnalyzer
    from urh_b200.signalprocessing.Signal import Signal

    noise = None

    def chain():
        s = Signal("", "bench")
        s.iq_array = IQArray(iq, skip_conversion=True)
        s.noise_threshold = noise
        s.auto_detect()
        pa = ProtocolAnalyzer(s)
        pa.get_protocol_from_signal()
        return [(m.plain_bits_str, m.pause) for m in pa.messages]

    def noise_step():
        nonlocal noise
        noise = AI.detect_noise_level_iq(iq)
        return noise

    return [("detect_noise_level_iq", noise_step),
            ("segment_messages_iq", lambda: AI.segment_messages_iq(iq, noise)),
            ("estimate", lambda: AI.estimate(IQArray(iq, skip_conversion=True))),
            ("signal_chain", chain)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=30)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--huge", action="store_true")
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.device import PinnedArray

    ctx = _lib.default_context()
    info = {"card": card(), "device": ctx.device_info()["name"], "log2n": args.log2n, "runs": args.runs, "results": []}
    print(json.dumps({"card": info["card"]}), flush=True)
    n = 1 << args.log2n
    for dtype in (np.float32, np.int8):
        buf = PinnedArray((n, 2), dtype)
        fill(buf.array)
        iq = buf.array
        names = [name for name, _ in steps(iq)]
        best = {(m, k): float("inf") for m in ("stream", "resident") for k in names}
        outs = {}
        for r in range(args.runs + 1):
            for mode in ("stream", "resident"):
                if mode == "stream":
                    os.environ["URH_B200_DEVICE_BUDGET"] = str(1 << 20)
                else:
                    os.environ.pop("URH_B200_DEVICE_BUDGET", None)
                for name, fn in steps(iq):
                    dt, out = timed(fn)
                    outs[(mode, name)] = out
                    if r > 0:
                        best[(mode, name)] = min(best[(mode, name)], dt)
        os.environ.pop("URH_B200_DEVICE_BUDGET", None)
        for name in names:
            row = {"dtype": np.dtype(dtype).name, "step": name, "stream_s": best[("stream", name)], "resident_s": best[("resident", name)],
                   "gb_per_s_stream": n * iq.itemsize * 2 / best[("stream", name)] / 1e9,
                   "parity": outs[("stream", name)] == outs[("resident", name)]}
            info["results"].append(row)
            print(json.dumps(row), flush=True)
        buf.free()
    info["huge"] = "not run"
    if args.huge:
        from urh_b200.ainterpretation import AutoInterpretation as AI

        total = ctx.device_info()["total_mem"]
        nh = (total // 8 + (1 << 30))
        try:
            buf = PinnedArray((nh, 2), np.float32)
        except (MemoryError, RuntimeError) as e:
            info["huge"] = "not run: %s" % e
        else:
            fill(buf.array)
            dt, est = timed(lambda: AI.estimate(buf.array))
            info["huge"] = {"samples": nh, "estimate_s": dt, "estimate": repr(est)}
            buf.free()
        print(json.dumps({"huge": info["huge"]}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1, default=str)


if __name__ == "__main__":
    main()
