#!/usr/bin/env python
"""BASELINE.json configs[2] and configs[3] end to end on one H100 (data resident in HBM, CUDA-event timing per stage).
One JSON object per line.

  configs[2]: 256 MiSample ASK capture -> FIR band-pass (101 taps) -> ASK demod -> spectrogram STFT(1024, hop 512)
  configs[3]: GFSK Modulator.modulate of 10 M random bits -> IQ -> FSK demod + digitize -> bits, bit-exact round trip

    python tools/bench_configs.py [--log2n 28] [--bits 10000000] > configs.jsonl

  --gpus N (under torchrun, one process per GPU): configs[2] on N GPUs with weak scaling, 2^log2n samples per rank, each rank
  modulating its own block.  Stages: halo exchange, band-pass, ASK demod + center + digitize, dB map; per stage the slowest rank's
  CUDA-event time.  edge_parity: at every shard edge rank 0 reruns the single-GPU kernels on +-2^16 samples (plus halos) fetched
  over NCCL and counts the band-pass and dB-map words that differ from the sharded ones (0 = bit-identical).

    torchrun --nproc-per-node 8 tools/bench_configs.py --gpus 8
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
    ap.add_argument("--gpus", type=int, default=0)
    args = ap.parse_args()
    if args.gpus:
        return sharded_config2(args)
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
                             "spectrogram dB (k_stft_r16)": ms_spec, "total": total},
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


def sharded_config2(args):
    import torch.distributed as dist

    if "RANK" not in os.environ and args.gpus == 1:   # one GPU needs no launcher
        os.environ.update(RANK="0", WORLD_SIZE="1", MASTER_ADDR="127.0.0.1", MASTER_PORT="29561")
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    if world != args.gpus:
        raise SystemExit("--gpus %d but %d ranks: launch with torchrun --nproc-per-node %d" % (args.gpus, world, args.gpus))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from urh_b200 import _lib, dist as udist
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Filter import Filter

    ctx = _lib.default_context(int(os.environ.get("LOCAL_RANK", rank)))
    lib = ctx.lib
    hx = udist.HostExchange()
    udist.init_nccl(ctx, hx)
    sps, W, hop, edge = 100, 1024, 512, 1 << 16
    bits = np.random.default_rng(1 + rank).integers(0, 2, (1 << args.log2n) // sps).astype(np.uint8)
    d_cap, off = sf.modulate_batch([bits], sps, "ASK", np.array([0.1, 1.0], np.float32), 1, 1.0, 0.05 * 2e6, 0.0, 2e6, 0, 0, np.float32,
                                   device_result=True)
    n_local = int(off[-1])
    sizes = hx.allgather(n_local)
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    bounds = [(int(starts[q]), int(starts[q + 1])) for q in range(world)]
    n = bounds[-1][1]
    g0 = bounds[rank][0]
    h = Filter.bandpass_taps(0.03, 0.07, Filter.get_bandwidth_from_filter_length(101))
    plan = udist.bandpass_plan(n, len(h), bounds)
    left, right, offset = plan[rank]
    sb = udist.ShardBuffer(ctx, n_local, np.float32, halo=left, right=right)
    ctx.check(lib.urh_memcpy_d2d(ctx.handle, C.c_void_p(sb.shard.ptr), C.c_void_p(d_cap.ptr), sb.shard.nbytes))
    d_cap.free()
    d_t = to_device(np.ascontiguousarray(h, dtype=np.complex128).view(np.float64), ctx)
    filt = udist.ShardBuffer(ctx, n_local, np.float32, halo=1)
    d_qad = DeviceArray(ctx, (n_local,), np.float32)
    win = sb.window(left, right)
    ms = {}

    def stage(name, fn):
        ctx.sync()
        hx.barrier()
        ctx.timer_start()
        out = fn()
        ms[name] = ctx.timer_stop()
        return out

    def bandpass():
        ctx.check(lib.urh_convolve_c128(ctx.handle, C.c_void_p(win.ptr), len(win), C.c_void_p(d_t.ptr), len(h), int(offset), n_local,
                                        C.c_void_p(filt.shard.ptr)))
        udist.exchange_halos(ctx, hx, filt, [(1 if q else 0, 0) for q in range(world)])

    for _ in range(2):   # the first round warms up NCCL, cuFFT plans and the module loads
        stage("halo exchange", lambda: udist.exchange_halos(ctx, hx, sb, [(a, b) for a, b, _ in plan]))
        stage("band-pass (101 taps, complex128, double accumulation)", bandpass)
        center, rows = stage("ASK demod + center + digitize", lambda: udist.demod_center_digitize_distributed(
            ctx, rank, world, filt, g0, n, 0.05, "ASK", 5, sps, d_qad, fetch=False))
        f0, db = stage("dB map STFT(1024, hop 512)", lambda: udist.spectrogram_db_sharded(ctx, hx, filt, bounds, W, 0.5))
    worst = {k: max(v[k] for v in hx.allgather(ms)) for k in ms}
    # edge parity: the single-GPU kernels on a window around every shard edge against the sharded words
    frames = hx.allgather((f0, len(db)))
    fbounds = [(a, a + c) for a, c in frames]
    half = (len(h) - 1) // 2
    d_w = to_device(np.hanning(W), ctx)
    diff = 0
    for e in starts[1:-1]:
        ka, kb = max(0, int(e) - edge), min(n, int(e) + edge)
        ra, rb = max(0, ka - half), min(n, kb + half)
        raw = udist.fetch_range(ctx, rank, bounds, sb.shard, ra, rb, 0)
        got = udist.fetch_range(ctx, rank, bounds, filt.shard, ka, kb, 0)
        fa, fb = -(-ka // hop), (kb - W) // hop + 1
        got_db = udist.fetch_range(ctx, rank, fbounds, db, fa, fb, 0)
        if rank == 0:
            ref = DeviceArray(ctx, (kb - ka, 2), np.float32)
            ctx.check(lib.urh_convolve_c128(ctx.handle, C.c_void_p(raw.ptr), rb - ra, C.c_void_p(d_t.ptr), len(h), ka - ra + half, kb - ka,
                                            C.c_void_p(ref.ptr)))
            ref_db = DeviceArray(ctx, (fb - fa, W), np.float32)
            src = ref[fa * hop - ka:]
            ctx.check(lib.urh_spectrogram_db(ctx.handle, C.c_void_p(src.ptr), len(src), W, hop, C.c_void_p(d_w.ptr), fb - fa, C.c_void_p(ref_db.ptr)))
            diff += int((got.get().view(np.uint32) != ref.get().view(np.uint32)).sum())
            diff += int((got_db.get().view(np.uint32) != ref_db.get().view(np.uint32)).sum())
    if rank == 0:
        total = sum(worst.values())
        print(json.dumps({"config": "configs[2] sharded: ASK capture -> 101-tap band-pass -> ASK demod+center+digitize -> STFT(1024, hop 512) dB",
                          "gpus": world, "samples_per_rank": n_local, "samples": n, "ms_max_over_ranks": worst, "total_ms": total,
                          "MSamples_per_s": n / total / 1e3, "center": center, "edge_parity": diff}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
