"""GPU (>= 2 devices): the sharded band-pass, FIR, DC correction, dB map and spectrogram images (urh_b200.dist, NCCL halos) equal the
single-GPU public functions bit for bit.  Skipped on a 1-GPU box."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_filters_and_spectrogram_match_single_gpu():
    from urh_b200 import _lib

    n = _lib.load_library().urh_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "dist_filter_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert "DIST_FILTER_RESULT OK" in out.stdout, out.stdout[-3000:]
