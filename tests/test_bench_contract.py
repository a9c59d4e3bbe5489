"""CPU: the parts of bench.py's contract that need no GPU - the reference arm's JSON line (the reference's own kernels on the host
cores, keys the driver reads) and the per-block structure of the synthetic capture (equal work per GPU at every N)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_line():
    # without oracle/_ref the arm times the C oracle port ("kind": "port"), which build() always compiles
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                          "--cpu-log2n", "18"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"].startswith("MSamples/s") and d["unit"] == "MSamples/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["gpu_launches"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["steps"] == 1 and cb["sample"].endswith("median of 1")                 # --steps sets the timed steps of this arm too
    e = d["e2e"]
    assert e["value"] == d["value"] and e["unit"] == d["unit"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0
    assert d["config"]["workload"].startswith("2-FSK complex64")


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith("{")]


def test_capture_blocks_are_alike():
    sys.path.insert(0, ROOT)
    import bench

    n = 1 << 20
    base = bench.capture_gaps(n, 0)
    assert base == (int(0.40 * n), int(0.43 * n), int(0.97 * n))       # N = 1: the single-GPU capture of BASELINE configs[1]
    for rank in range(1, 8):
        g = bench.capture_gaps(n, rank)
        assert tuple(x - rank * n for x in g) == base                    # every block is built like the first
        assert rank * n <= g[0] < g[1] < g[2] < (rank + 1) * n


@pytest.mark.gpu
def test_dump_outputs_are_small_float_and_repeatable(tmp_path):
    """--dump-outputs: the last timed step's results as float32 / float64 .npy files under 64 MB, identical for identical inputs
    whatever the number of steps"""
    import numpy as np

    dirs = []
    for steps in (1, 3):
        d = tmp_path / ("steps%d" % steps)
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--log2n", "22", "--steps", str(steps), "--warmup", "1",
                              "--no-e2e", "--no-cpu", "--no-parity", "--dump-outputs", str(d)], capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert out.returncode == 0, out.stderr[-2000:]
        assert json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])["steps"] == steps
        dirs.append(d)
    names = sorted(p.name for p in dirs[0].iterdir())
    assert names == ["center.npy", "pulse_rows_count.npy", "pulse_rows_sample.npy", "pulse_rows_sample_index.npy", "qad_sample.npy",
                     "qad_sample_position.npy"]
    assert names == sorted(p.name for p in dirs[1].iterdir())
    assert sum((dirs[0] / f).stat().st_size for f in names) < 64 << 20
    for f in names:
        a, b = np.load(dirs[0] / f), np.load(dirs[1] / f)
        assert a.dtype in (np.float32, np.float64) and a.size > 0, f
        assert a.dtype == b.dtype and np.array_equal(a, b), f
