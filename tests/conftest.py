import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    d = {k: z[k] for k in z.files}
    if "meta" in d:
        d["meta"] = json.loads(str(d["meta"]))
    return d


CAPTURES = ["fsk", "ask", "ask_short", "psk_gen_noisy", "enocean", "FSK10", "homematic", "esaver", "two_participants"]


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o

    o.build()
    return o


@pytest.fixture(scope="session")
def ctx():
    from urh_b200 import _lib

    return _lib.default_context()


def bits_equal(a: np.ndarray, b: np.ndarray) -> int:
    """number of differing 32-bit words between two float32 arrays (NaN-safe, sign-of-zero aware)"""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    assert a.shape == b.shape, (a.shape, b.shape)
    return int((a.view(np.uint32) != b.view(np.uint32)).sum())


def synth_fsk(n, sps=100, seed=0, noise_sigma=0.01, gap_every=None, dtype=np.float32):
    """Seeded phase-continuous 2-FSK capture with AWGN and noise-only gaps (SURVEY §8d recipe, small)."""
    rng = np.random.default_rng(seed)
    nsym = n // sps + 1
    bits = rng.integers(0, 2, nsym)
    f = np.repeat(np.where(bits > 0, 0.01, -0.01), sps)[:n]
    phase = 2 * np.pi * np.cumsum(f)
    amp = np.ones(n)
    if gap_every:
        for s in range(gap_every, n, 2 * gap_every):
            amp[s: s + gap_every // 2] = 0.0
    x = amp * np.exp(1j * phase) + noise_sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    iq = np.empty((n, 2), dtype=np.float32)
    iq[:, 0] = x.real
    iq[:, 1] = x.imag
    if dtype == np.float32:
        return iq
    if dtype == np.int8:
        return np.clip(iq * 100, -128, 127).astype(np.int8)
    if dtype == np.uint8:
        return np.clip(iq * 100 + 128, 0, 255).astype(np.uint8)
    if dtype == np.int16:
        return np.clip(iq * 20000, -32768, 32767).astype(np.int16)
    if dtype == np.uint16:
        return np.clip(iq * 20000 + 32768, 0, 65535).astype(np.uint16)
    raise ValueError(dtype)
