"""Float32 IQ captures with infinite, NaN, huge, subnormal and zero samples for the ASK/FSK demodulation tests.

tests/test_oracle.py pins the oracle's afp_demod to the reference on them; tests/test_gpu_dense_edges.py compares the kernels with
the oracle.  Every special value comes with every sign, after and before neighbours with zero and nonzero parts.  Results are
compared as words with NaN folded to one word: the NaN payload is not pinned (x86 gives 0xffc00000 or the input's payload, the
GPU 0x7fffffff)."""
import numpy as np

INF, NAN = float("inf"), float("nan")
FMAX = float(np.finfo(np.float32).max)
SUB = float(np.float32(1e-40))       # subnormal
TINY = float(np.float32(1.4e-45))    # the smallest subnormal

# first-quadrant magnitudes of the special samples; SPECIALS expands every sign
_BASE = [(0.5, INF), (0.3, INF), (INF, INF), (0.0, INF), (INF, 0.5), (INF, 0.0), (NAN, 0.5), (0.5, NAN), (NAN, INF), (INF, NAN),
         (1e30, 1e30), (FMAX, FMAX), (FMAX, 0.5), (3e38, 3e38), (SUB, SUB), (TINY, 0.5), (SUB, 1.0), (0.0, 0.0)]
SPECIALS = sorted({(float(np.copysign(re, sr)), float(np.copysign(im, si))) for re, im in _BASE for sr in (1, -1) for si in (1, -1)},
                  key=repr)
# neighbours: both parts nonzero, one part zero, both zero, a subnormal part
NEIGHBOURS = [(1.0, 1.0), (1.0, -1.0), (0.7, 0.7), (0.3, 0.7), (-0.5, -0.25), (2.0, 0.0), (0.0, 1.0), (0.0, 0.0), (-0.0, -0.0),
              (SUB, 1.0)]


def folded(q):
    """the words of a float32 result with every NaN folded to 0x7fc00000"""
    q = np.asarray(q, dtype=np.float32)
    w = q.view(np.uint32).copy()
    w[np.isnan(q)] = 0x7FC00000
    return w


def fsk_tone(n, seed, step=0.3):
    """unit-amplitude samples rotating by +-step rad (runs of 5..60 samples) from a phase where both parts stay far from zero"""
    rng = np.random.default_rng(seed)
    runs = rng.integers(5, 60, n // 5 + 1)
    sign = np.repeat(np.where(np.arange(len(runs)) % 2 == 0, 1.0, -1.0), runs)[:n]
    ph = 0.4 + np.cumsum(sign * step)
    iq = np.stack([np.cos(ph), np.sin(ph)], axis=1).astype(np.float32)
    small = np.abs(iq) < 1e-3
    iq[small] = np.float32(1e-3)
    return iq


def pinned_captures():
    """(name, iq) float32 captures of a few thousand samples: every special after and before every neighbour, and specials in a row"""
    iq = fsk_tone(len(SPECIALS) * len(NEIGHBOURS) * 4 + 16, seed=3)
    pos = 8
    for j, v in enumerate(SPECIALS):
        for k, p in enumerate(NEIGHBOURS):
            iq[pos] = p
            iq[pos + 1] = v
            iq[pos + 2] = NEIGHBOURS[(k + 3 + j) % len(NEIGHBOURS)]
            pos += 4
    yield "after_before", iq
    rng = np.random.default_rng(5)
    iq = fsk_tone(4000, seed=4)
    idx = rng.integers(0, len(SPECIALS), 3000)
    at = 10 + np.sort(rng.choice(3980, 1500, replace=False))
    for a, i in zip(at, idx):
        iq[a] = SPECIALS[i]
    iq[at + 1] = [SPECIALS[i] for i in idx[1500:]]
    yield "in_a_row", iq


# the bug's cases, checked by value: (predecessor, sample) -> the reference's angle word
REFERENCE_TABLE = [
    ((1.0, 1.0), (0.5, INF), 0x3F490FDB),
    ((0.5, INF), (0.3, 0.7), 0xBF490FDB),
    ((1.0, -1.0), (-0.5, -INF), 0xBF490FDB),
    ((0.7, 0.7), (INF, INF), 0x3F490FDB),
    ((1.0, 1.0), (0.0, -INF), 0xC016CBE4),
]
