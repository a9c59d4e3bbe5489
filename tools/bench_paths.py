#!/usr/bin/env python
"""Secondary measurements (not the headline bench): every other row of the scope table with data resident in HBM,
CUDA-event timing, algorithmic bytes per SURVEY §8d.  Writes one JSON object per line.

    python tools/bench_paths.py [--log2n 26] > secondary.jsonl
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


def timed(ctx, fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    ctx.sync()
    ts = []
    for _ in range(reps):
        ctx.timer_start()
        fn()
        ts.append(ctx.timer_stop())
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=26)
    args = ap.parse_args()
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.cythonext import signal_functions as sf, util, auto_interpretation as cai
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.signalprocessing.Spectrogram import Spectrogram
    from conftest import synth_fsk
    from test_gpu_costas import synth_psk

    ctx = _lib.default_context()
    lib = ctx.lib
    n = 1 << args.log2n
    peak = 3350.0   # H100 SXM data sheet (HBM3), unless MEASURED_PEAKS.json gives a measured figure
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass

    def emit(name, ms, samples, bytes_per_sample=None, note=""):
        rec = {"path": name, "samples": int(samples), "ms": ms, "MSamples_per_s": samples / ms / 1e3}
        if bytes_per_sample:
            rec["algorithmic_B_per_sample"] = bytes_per_sample
            rec["GB_per_s"] = samples * bytes_per_sample / ms / 1e6
            rec["frac_of_hbm_peak"] = rec["GB_per_s"] / peak
        if note:
            rec["note"] = note
        print(json.dumps(rec), flush=True)

    # synthetic FSK capture (same recipe as bench.py) generated in HBM
    sys.path.insert(0, ROOT)
    import bench as B

    nsym = n // B.SPS + 2
    b, s = B.make_symbols(nsym, seed=5)
    d_b = DeviceArray(ctx, (nsym,), np.int8).set(b)
    d_s = DeviceArray(ctx, (nsym,), np.int32).set(s)
    d_iq = DeviceArray(ctx, (n, 2), np.float32)
    ctx.check(lib.urh_synth_fsk(ctx.handle, C.c_void_p(d_iq.ptr), n, 0, B.SPS, C.c_void_p(d_b.ptr), C.c_void_p(d_s.ptr),
                                C.c_double(B.FDEV / B.FS), 1.0, B.SIGMA, 99, 6_000_000, 5_000_000, int(0.40 * n), int(0.43 * n), int(0.97 * n)))
    ctx.sync()

    # the SDR-native sample formats (2^26-sample slice of the same capture, scaled to the integer range)
    ni = min(n, 1 << 26)
    host = d_iq[:ni].get()
    for dt, scale, noise in ((np.int16, 8000.0, B.NOISE_MAG * 8000.0), (np.int8, 100.0, B.NOISE_MAG * 100.0)):
        d_i = to_device(np.ascontiguousarray(np.round(host * scale).astype(dt)), ctx)
        d_qi = DeviceArray(ctx, (ni,), np.float32)
        k = C.c_int64(0)
        run = lambda: ctx.check(lib.urh_demod_digitize(ctx.handle, C.c_void_p(d_i.ptr), _lib.dtype_code(dt), ni, float(noise), _lib.MOD_FSK, 0.0, 5, B.SPS, 1,
                                                       0.1, C.c_void_p(d_qi.ptr), C.byref(k)))
        emit("demod + digitize FSK, %s capture (fused, center given)" % np.dtype(dt).name, timed(ctx, run), ni, 2 * np.dtype(dt).itemsize + 4)
        del d_i, d_qi
    del host
    q = sf.afp_demod(d_iq, B.NOISE_MAG, "FSK", 2)
    emit("afp_demod FSK (exact, no digitizer)", timed(ctx, lambda: sf.afp_demod(d_iq, B.NOISE_MAG, "FSK", 2)), n, 12)
    emit("afp_demod ASK", timed(ctx, lambda: sf.afp_demod(d_iq, B.NOISE_MAG, "ASK", 2)), n, 12)
    emit("grab_pulse_lens (stand-alone, qad in HBM)", timed(ctx, lambda: sf.grab_pulse_lens(q, 0.0, 5, "FSK", 100)), n, 4, "incl. D2H of the pulse table")
    emit("detect_noise_level from IQ (no float64 magnitudes)", timed(ctx, lambda: AI.detect_noise_level_iq(d_iq)), n, 8)
    emit("detect_center stand-alone (tile statistics pass + histogram pass over qad)", timed(ctx, lambda: AI.detect_center(q)), n, 8, "incl. host peak picking")
    mags = util.get_magnitudes(d_iq)
    emit("get_magnitudes (float64 out)", timed(ctx, lambda: util.get_magnitudes(d_iq)), n, 16)
    emit("segment_messages_from_magnitudes (float64 in)", timed(ctx, lambda: cai.segment_messages_from_magnitudes(mags, B.NOISE_MAG)), n, 8)
    del mags

    # PSK (speculative Costas)
    npsk = min(n, 1 << 24)
    iqp = to_device(synth_psk(npsk, 2, seed=3), ctx)
    ms = timed(ctx, lambda: sf.afp_demod(iqp, 0.2, "PSK", 2), reps=3, warm=1)
    st = (C.c_int64 * 3)()
    lib.urh_costas_stats(ctx.handle, st)
    emit("afp_demod PSK order 2 (speculative Costas, bit-exact)", ms, npsk, 12, "chunks fast/slow/samples stepped = %s" % list(st))
    iqp4 = to_device(synth_psk(npsk, 4, seed=4), ctx)
    emit("afp_demod PSK order 4 (speculative Costas, bit-exact)", timed(ctx, lambda: sf.afp_demod(iqp4, 0.2, "PSK", 4), reps=3, warm=1), npsk, 12)
    del iqp, iqp4

    # filters / spectrogram on a 2^24 complex64 capture
    nf = min(n, 1 << 24)
    x = d_iq[:nf]
    xc = DeviceArray(ctx, (nf,), np.complex64, ptr=x.ptr, base=x)
    taps = (np.random.default_rng(0).standard_normal(101) + 1j * np.random.default_rng(1).standard_normal(101)).astype(np.complex64)
    ms = timed(ctx, lambda: sf.fir_filter(xc, taps), reps=3, warm=1)
    emit("fir_filter 101 complex taps (exact order)", ms, nf, 16, "FP32-ALU-bound: %.1f unfused GFLOP/s" % (nf * 808 / ms / 1e6))
    d_t = to_device(np.ascontiguousarray(taps.astype(np.complex128)).view(np.float64), ctx)
    out = DeviceArray(ctx, (nf,), np.complex64)
    ms = timed(ctx, lambda: ctx.check(lib.urh_convolve_c128(ctx.handle, C.c_void_p(xc.ptr), nf, C.c_void_p(d_t.ptr), 101, 50, nf, C.c_void_p(out.ptr))), reps=3, warm=1)
    emit("band-pass convolution 101 complex128 taps (double accumulation)", ms, nf, 16)
    out2 = DeviceArray(ctx, (nf, 2), np.float32)
    emit("DC correction (double reduction path)", timed(ctx, lambda: ctx.check(lib.urh_dc_correction(ctx.handle, C.c_void_p(x.ptr), nf, C.c_void_p(out2.ptr), 0))), nf, 24)
    W, hop = 1024, 512
    frames = (nf - W) // hop + 1
    d_w = to_device(np.hanning(W), ctx)
    d_db = DeviceArray(ctx, (frames, W), np.float32)
    ms = timed(ctx, lambda: ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(x.ptr), nf, W, hop, C.c_void_p(d_w.ptr), frames, C.c_void_p(d_db.ptr))), reps=3, warm=1)
    emit("spectrogram STFT(1024, hop 512, Z2Z) -> dB", ms, nf, 16)

    # modulator: 10 000 messages x 1000 bits (config 4 shape), GFSK and FSK, float32
    rng = np.random.default_rng(2)
    msgs = rng.integers(0, 2, (2000, 1000), dtype=np.uint8)   # rectangular batch: no per-message host work (tools/bench_modulate.py
    for mt, params in (("FSK", [-20e3, 20e3]), ("GFSK", [-20e3, 20e3]), ("PSK", [-1.5, 1.5])):   # separates stream time from wall time)
        t0 = time.perf_counter()
        d_out, off = sf.modulate_batch(msgs, 100, mt, np.array(params, np.float32), 1, 1.0, 0.0, 0.0, 2e6, 0, 0, np.float32, device_result=True)
        ctx.sync()
        t1 = time.perf_counter()
        d_out, off = sf.modulate_batch(msgs, 100, mt, np.array(params, np.float32), 1, 1.0, 0.0, 0.0, 2e6, 0, 0, np.float32, device_result=True)
        ctx.sync()
        ms = (time.perf_counter() - t1) * 1e3
        emit("modulate_batch %s 2000 msgs x 1000 bits x 100 sps (result in HBM)" % mt, ms, int(off[-1]), 8, "wall clock incl. host prep")


if __name__ == "__main__":
    main()
