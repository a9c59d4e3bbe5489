"""GPU (>= 2 devices): sharded capture over NCCL == single-GPU result.  Skipped on a 1-GPU box.

tests/test_gpu_dist_one_gpu.py runs the noise level, segmentation, center protocol, sharded Costas loop, estimate() and halo paths
rank by rank on one GPU with host stand-ins for the NCCL calls dist.py makes from Python.  What only this test covers is NCCL itself and the
exchanges the library makes from C: the sharded digitizer (urh_shard_digitize), the fused demod + center + digitize step
(urh_shard_demod_center_digitize) and the center chain's rank/world mode."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_capture_matches_single_gpu():
    from urh_b200 import _lib

    n = _lib.load_library().urh_device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "dist_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert "DIST_GPU_RESULT OK" in out.stdout, out.stdout[-3000:]
