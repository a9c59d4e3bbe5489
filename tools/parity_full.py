#!/usr/bin/env python
"""Full-size parity run (SURVEY §8d, config 2): the bench's 2^30-sample synthetic capture through the CUDA path and through
the CPU oracle (C restatement / reference build, all host threads), compared bit for bit:
  * qad of afp_demod FSK: uint32 view equal everywhere
  * the pulse table of grab_pulse_lens for the DETECTED center (and for center 0, tolerance 0 and 5)
  * detect_center within 2e-6
Needs ~30 GB of host memory and a minute or two of CPU time at 2^30; not part of the pytest suite.

    python tools/parity_full.py [--log2n 30] > parity_full.json
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
    ap.add_argument("--log2n", type=int, default=30)
    args = ap.parse_args()
    import bench as B
    from oracle import oracle
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray
    from urh_b200.cythonext import signal_functions as sf

    os.environ["OMP_NUM_THREADS"] = str(os.cpu_count() or 1)
    ctx = _lib.default_context()
    lib = ctx.lib
    n = 1 << args.log2n
    nsym = n // B.SPS + 2
    b, s = B.make_symbols(nsym, seed=1000)
    d_b = DeviceArray(ctx, (nsym,), np.int8).set(b)
    d_s = DeviceArray(ctx, (nsym,), np.int32).set(s)
    d_iq = DeviceArray(ctx, (n, 2), np.float32)
    ctx.check(lib.urh_synth_fsk(ctx.handle, C.c_void_p(d_iq.ptr), n, 0, B.SPS, C.c_void_p(d_b.ptr), C.c_void_p(d_s.ptr),
                                C.c_double(B.FDEV / B.FS), 1.0, B.SIGMA, 12345, 6_000_000, 5_000_000,
                                int(0.40 * n), int(0.43 * n), int(0.97 * n)))
    ctx.sync()
    out = {"samples": n, "checks": {}}
    center, rows, qad = sf.demod_center_digitize(d_iq, B.NOISE_MAG, "FSK", B.TOL, B.SPS, return_qad=True)
    q_gpu = qad.get()
    iq = d_iq.get()
    t0 = time.time()
    q_ref = oracle.afp_demod(iq, B.NOISE_MAG, "FSK", 2)
    out["oracle_demod_s"] = time.time() - t0
    out["checks"]["qad_words_differing"] = int(np.count_nonzero(q_gpu.view(np.uint32) != q_ref.view(np.uint32)))
    del iq
    t0 = time.time()
    c_ref = oracle.detect_center(q_ref)
    out["oracle_center_s"] = time.time() - t0
    out["center_gpu"], out["center_oracle"] = center, c_ref
    out["checks"]["center_within_2e-6"] = bool(center is not None and c_ref is not None and abs(center - c_ref) <= 2e-6 * max(1.0, abs(c_ref)))
    t0 = time.time()
    r_ref = oracle.grab_pulse_lens(q_ref, center, B.TOL, "FSK", B.SPS)
    out["oracle_digitize_s"] = time.time() - t0
    out["pulse_rows"] = int(len(rows))
    out["checks"]["rows_equal_detected_center"] = bool(np.array_equal(rows, r_ref))
    for c, tol in ((0.0, 0), (0.0, 5)):
        r_gpu = sf.grab_pulse_lens(qad, c, tol, "FSK", B.SPS)
        out["checks"]["rows_equal_center%g_tol%d" % (c, tol)] = bool(np.array_equal(r_gpu, oracle.grab_pulse_lens(q_ref, c, tol, "FSK", B.SPS)))
    _, r_fused = sf.demod_digitize(d_iq, B.NOISE_MAG, "FSK", 0.0, B.TOL, B.SPS, return_qad=False)
    out["checks"]["fused_rows_equal_center0_tol5"] = bool(np.array_equal(r_fused, oracle.grab_pulse_lens(q_ref, 0.0, B.TOL, "FSK", B.SPS)))
    out["all_ok"] = all(v is True or v == 0 for v in out["checks"].values())
    print(json.dumps(out))
    return 0 if out["all_ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
