#!/usr/bin/env python
"""BASELINE.json configs[2] and configs[3] end to end on one H100 (data resident in HBM, CUDA-event timing per stage).
One JSON object per line.

  configs[2]: 256 MiSample ASK capture -> FIR band-pass (101 taps) -> ASK demod -> spectrogram STFT(1024, hop 512)
  configs[3]: GFSK Modulator.modulate of 10 M random bits -> IQ -> FSK demod + digitize -> bits, bit-exact round trip

    python tools/bench_configs.py [--log2n 28] [--bits 10000000] > configs.jsonl
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=28)
    ap.add_argument("--bits", type=int, default=10_000_000)
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Filter import Filter

    ctx = _lib.default_context()
    lib = ctx.lib

    def timed(fn, reps=3, warm=1):
        for _ in range(warm):
            fn()
        ctx.sync()
        ts = []
        for _ in range(reps):
            ctx.timer_start()
            fn()
            ts.append(ctx.timer_stop())
        return float(np.median(ts))

    # ---------------- configs[2] --------------------------------------------------------------------------------
    n = 1 << args.log2n
    sps = 100
    rng = np.random.default_rng(1)
    nbits = n // sps
    bits = rng.integers(0, 2, nbits).astype(np.uint8)
    # OOK/ASK capture at carrier +0.05 fs, produced by the modulator kernel directly in HBM
    d_cap, off = sf.modulate_batch([bits], sps, "ASK", np.array([0.1, 1.0], np.float32), 1, 1.0, 0.05 * 2e6, 0.0, 2e6, 0,
                                   0, np.float32, device_result=True)
    n2 = int(off[-1])
    h = Filter.design_windowed_sinc_bandpass(0.03, 0.07, Filter.get_bandwidth_from_filter_length(101))
    assert len(h) == 101, len(h)
    d_t = to_device(np.ascontiguousarray(h.astype(np.complex128)).view(np.float64), ctx)
    d_filt = DeviceArray(ctx, (n2, 2), np.float32)
    ms_fir = timed(lambda: ctx.check(lib.urh_convolve_c128(ctx.handle, C.c_void_p(d_cap.ptr), n2, C.c_void_p(d_t.ptr), 101, 50, n2,
                                                           C.c_void_p(d_filt.ptr))))
    d_qad = DeviceArray(ctx, (n2,), np.float32)
    ms_demod = timed(lambda: ctx.check(lib.urh_afp_demod(ctx.handle, C.c_void_p(d_filt.ptr), _lib.DT_F32, n2, 0.05, _lib.MOD_ASK, 2, 0.1,
                                                         C.c_void_p(d_qad.ptr))))
    W, hop = 1024, 512
    frames = (n2 - W) // hop + 1
    d_w = to_device(np.hanning(W), ctx)
    d_db = DeviceArray(ctx, (frames, W), np.float32)
    ms_spec = timed(lambda: ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_filt.ptr), n2, W, hop, C.c_void_p(d_w.ptr), frames,
                                                             C.c_void_p(d_db.ptr))))
    # sanity: the band-pass keeps the carrier, the demodulated envelope follows the bits
    q = d_qad[: 50 * sps].get()
    env = q.reshape(-1, sps)[:, sps // 2] > 0.3
    ok2 = bool(np.array_equal(env.astype(np.uint8), bits[:50]))
    total = ms_fir + ms_demod + ms_spec
    print(json.dumps({"config": "configs[2]: ASK capture -> 101-tap band-pass -> ASK demod -> STFT(1024, hop 512) dB", "samples": n2,
                      "ms": {"band-pass (complex128 taps, double accumulation)": ms_fir, "afp_demod ASK": ms_demod,
                             "spectrogram dB (cuFFT Z2Z)": ms_spec, "total": total},
                      "MSamples_per_s": n2 / total / 1e3, "envelope_matches_bits": ok2}), flush=True)
    del d_cap, d_filt, d_qad, d_db

    # ---------------- configs[3] --------------------------------------------------------------------------------
    # The reference computes t = i / sample_rate and the GFSK phases in float32, so ONE 10 Mbit message (10^9 samples) has no
    # meaningful phase in either implementation; URH modulates message by message.  10 Mbit = nmsg messages x 1000 bits.
    per = 1000
    nmsg = args.bits // per
    bits = rng.integers(0, 2, (nmsg, per)).astype(np.uint8)
    params = np.array([-20e3, 20e3], np.float32)
    pause = 2000                        # 20 symbols of silence: a message separator (pause_threshold 8)
    d_iq, off = sf.modulate_batch(bits, sps, "GFSK", params, 1, 1.0, 0.0, 0.0, 2e6, pause, 0, np.float32, device_result=True)
    ctx.sync()
    ns = int(off[-1])
    del d_iq
    t0 = time.perf_counter()
    d_iq, off = sf.modulate_batch(bits, sps, "GFSK", params, 1, 1.0, 0.0, 0.0, 2e6, pause, 0, np.float32, device_result=True)
    ctx.sync()
    wall_mod = (time.perf_counter() - t0) * 1e3
    k = C.c_int64(0)

    def demod():
        ctx.check(lib.urh_demod_digitize(ctx.handle, C.c_void_p(d_iq.ptr), _lib.DT_F32, ns, 0.05, _lib.MOD_FSK, 0.0, 5, sps, 1, 0.1, None,
                                         C.byref(k)))
    ms_dd = timed(demod)
    m, b, p = C.c_int64(0), C.c_int64(0), C.c_int64(0)

    def tobits():
        ctx.check(lib.urh_ppseq_to_bits(ctx.handle, None, k.value, sps, 1, 8, 0, C.byref(m), C.byref(b), C.byref(p)))
    ms_both = timed(lambda: (demod(), tobits()))
    demod()
    got, moff, pauses, _ = sf.ppseq_to_bits(int(k.value), sps, 1, write_bit_sample_pos=False)
    lens = np.diff(moff)
    same = len(pauses) == nmsg and bool(np.all(lens == per)) and bool(np.array_equal(got.reshape(nmsg, per), bits))
    bad = -1
    if not same and len(pauses) == nmsg:
        bad = int(sum(1 for q in range(nmsg) if lens[q] != per or not np.array_equal(got[moff[q]:moff[q + 1]], bits[q])))
    print(json.dumps({"config": "configs[3]: GFSK modulate %d x %d random bits (sps 100, BT 0.5, 2000-sample pauses) -> FSK demod+digitize -> bits"
                                % (nmsg, per), "samples": ns,
                      "ms": {"modulate_batch (wall, incl. host prep + H2D of the bits)": wall_mod, "demod+digitize (fused)": ms_dd,
                             "pulse table -> bits (device)": ms_both - ms_dd},
                      "pulse_rows": int(k.value), "messages": int(len(pauses)), "bits_recovered": int(len(got)),
                      "round_trip_bit_exact": same, "messages_differing": bad,
                      "MSamples_per_s_demod": ns / ms_dd / 1e3, "Mbit_per_s_modulate": nmsg * per / wall_mod / 1e3}), flush=True)


if __name__ == "__main__":
    main()
