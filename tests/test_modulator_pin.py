"""CPU suite: the oracle's modulator (urh_oracle.c: oracle_modulate) pinned word for word to the reference's compiled modulate_c
over a random matrix of ASK / FSK / PSK / OQPSK parameters; numpy's float32 arange fill (the GFSK time base) pinned as a rule; the
host build of glibc_sincosf.h pinned to libm at |x| >= 120 (the large-argument reduction only the modulator reaches).

The matrix (modulator_cases) and the libm harness are shared with tests/test_gpu_modulator_exact.py, which holds the GPU
modulator to the oracle on the same cases."""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODS = ("ASK", "FSK", "PSK", "OQPSK")
DTYPES = (np.int8, np.int16, np.float32)
SPS = (1, 2, 3, 7, 100, 1000)
STARTS = (0, 1, 5, 2 ** 24 - 1, 2 ** 24 + 1, 2 ** 31 + 1, 2 ** 32 - 1)
RATES = (1.0, 44100.0, 1e6, 2e6, 3e6)


def modulator_cases(n=420, max_samples=60_000):
    """Seeded modulate_c argument tuples (bits, sps, mod, params, bps, a, fc, phi, fs, pause, start, dtype) cycling every
    modulation, dtype, bps 1-8 (OQPSK: 2), sps, start and sample rate of the lists above.  Frequencies are negative and above
    Nyquist, one case in four on a MHz scale whatever the sample rate (at fs = 1 Hz and a large start the FSK correction term
    passes 1e15); ASK parameters include 0; bit counts are not always a multiple of bps; bits come uniform, in long runs or
    alternating.

    Left out because the reference itself is undefined there: OQPSK with fewer than 2 bits (its zeroing loop writes before the
    array), and amplitudes that push I/Q outside int32 (the float -> int conversion is undefined behaviour in C)."""
    rng = np.random.default_rng(2024)
    for k in range(n):
        mod, dt = MODS[k % 4], DTYPES[(k // 4) % 3]
        sps, start, fs = SPS[k % 6], STARTS[k % 7], RATES[k % 5]
        bps = 2 if mod == "OQPSK" else 1 + (k // 3) % 8
        nsym = int(rng.integers(1, max(2, min(3000, max_samples // sps)) + 1))
        nbits = nsym * bps + int(rng.integers(0, bps))
        style = k % 3
        if style == 0:
            bits = rng.integers(0, 2, nbits)
        elif style == 1:   # long runs of equal symbols
            bits = np.repeat(rng.integers(0, 2, nbits // 37 + 1), 37)[:nbits]
        else:              # alternating symbols
            sym = np.where(np.arange(nsym + 1) % 2 == 0, 0, (1 << bps) - 1)
            bits = ((sym[:, None] >> np.arange(bps - 1, -1, -1)) & 1).reshape(-1)[:nbits]
        bits = np.ascontiguousarray(bits, dtype=np.uint8)
        if mod == "OQPSK" and len(bits) < 2:
            bits = np.array([1, 0], np.uint8)
        fscale = 1e6 if (k // 4) % 4 == 1 else fs
        if dt == np.float32:
            a = float(np.float32(rng.uniform(0.05, 1.0)))
        else:   # the dtype's full scale, or well past it (C truncation wraps int8 / int16), I/Q inside int32
            a = float(np.iinfo(dt).max) * (float(rng.uniform(0.1, 1.0)) if k % 5 else float(rng.uniform(1.0, 3000.0)))
        m = 1 << bps
        if mod == "ASK":
            p = rng.uniform(0, a, m)
            p[rng.integers(0, m)] = 0.0
            if m > 2:
                p[rng.integers(0, m)] = 0.0
        elif mod == "FSK":
            p = fscale * rng.uniform(-1.5, 1.5, m)
            if m > 2:
                p[1] = p[0]   # two symbols with one frequency: no correction between them
        else:
            p = rng.uniform(-2 * np.pi, 2 * np.pi, m)
        fc = float(np.float32(fscale * rng.uniform(-1.5, 1.5)))
        phi = float(np.float32(rng.uniform(-np.pi, np.pi)))
        pause = int(rng.integers(0, 40))
        yield bits, sps, mod, np.asarray(p, np.float32), bps, a, fc, phi, fs, pause, start, dt


def mod_words(out):
    """a modulate_c result as integers: float32 samples as their bit patterns with NaN folded to one word (its payload is not
    pinned), integer samples as they are"""
    out = np.asarray(out)
    if out.dtype != np.float32:
        return out.astype(np.int64)
    w = out.view(np.uint32).astype(np.int64)
    w[np.isnan(out)] = 0x7FC00000
    return w


def test_oracle_modulator_pinned_to_reference(oracle, request):
    """oracle.modulate_c against the reference's compiled modulate_c on modulator_cases(), word for word.  The reference's
    answers are recorded in tests/golden/ref_modulator.json, so the pin also runs without the reference; with oracle/_ref built
    it also runs live.  GFSK is not pinned here: the reference's float32 np.convolve runs through OpenBLAS sdot, whose
    summation order depends on the host CPU."""
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, same

    c = Cassette("modulator", request.node.name)
    sf = ref_loader.load_kernels()[0] if (RECORD or ref_loader.kernels_available()) else None
    cases = 0
    for bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt in modulator_cases():
        mine = oracle.modulate_c(bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt)
        ref = lambda: np.asarray(sf.modulate_c(bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt))   # noqa: E731
        want = c.want(lambda: mod_words(ref()))
        where = (cases, mod, np.dtype(dt).name, sps, bps, len(bits), start, fs)
        assert mine.dtype == np.dtype(dt) and mine.shape == (len(bits) // bps * sps + pause, 2), where
        assert same(mod_words(mine), want), where
        if sf is not None:
            assert np.array_equal(mod_words(mine), mod_words(ref())), where
        cases += 1
    c.close()
    assert cases == 420


def arange_f32(start, n):
    """np.arange(start, start + n, dtype=np.float32) as numpy fills it: t0 = fl(start), t1 = fl(start + 1), d = fl(t1 - t0), then
    t_i = fl(t0 + fl(fl(i) * d)).  Not fl(start + i): from start = 1 they part at i = 2^24 + 1; at start = 2^31 + 1, d = 0."""
    t0, t1 = np.float32(start), np.float32(start + 1)
    d = np.float32(t1 - t0)
    return (t0 + np.arange(n, dtype=np.int64).astype(np.float32) * d).astype(np.float32)


def test_numpy_float32_arange_rule():
    """arange_f32 is numpy's own fill, word for word (the GFSK time base of the reference, signal_functions.pyx:210).  If numpy
    ever fills differently, this says so before the GPU test of the GFSK phases does."""
    chunk = 1 << 22
    for start, n in ((0, 2 ** 25 + 7), (1, 2 ** 25 + 7), (3, 2 ** 25 + 7), (5, 2 ** 24 + 9), (123457, 2 ** 25 + 7),
                     (2 ** 24 - 5, 2 ** 25 + 7), (2 ** 24 - 1, 10 ** 5), (2 ** 24 + 1, 10 ** 5), (2 ** 31 + 1, 10 ** 5),
                     (2 ** 32 - 3, 10 ** 5), (2 ** 32 - 1, 10 ** 5)):
        ref = np.arange(start, start + n, dtype=np.float32)
        for lo in range(0, n, chunk):
            hi = min(n, lo + chunk)
            want = ref[lo:hi]
            t0, d = np.float32(start), np.float32(np.float32(start + 1) - np.float32(start))
            mine = (t0 + np.arange(lo, hi, dtype=np.int64).astype(np.float32) * d).astype(np.float32)
            assert np.array_equal(mine.view(np.uint32), want.view(np.uint32)), (start, lo)
        assert np.array_equal(arange_f32(start, 1000).view(np.uint32), ref[:1000].view(np.uint32)), start
    # the rule is not fl(start + i)
    assert not np.array_equal(arange_f32(1, 2 ** 24 + 2), (np.arange(2 ** 24 + 2) + 1).astype(np.float32))
    assert np.all(arange_f32(2 ** 31 + 1, 1000) == np.float32(2 ** 31))


LIBM_HARNESS = r"""
#include <math.h>
#include "%s"
void restated(const float* y, float* sn, float* cs, int* ok, long n) {
    for (long i = 0; i < n; i++) urh_glibc_sincosf(y[i], &sn[i], &cs[i], &ok[i]);
}
void ref(const float* y, float* sn, float* cs, long n) {
    for (long i = 0; i < n; i++) { sn[i] = sinf(y[i]); cs[i] = cosf(y[i]); }
}
void ref_fmod_2pi(const double* v, double* out, long n) {
    for (long i = 0; i < n; i++) out[i] = fmod(v[i], 2.0 * M_PI);
}
/* the GFSK phase recurrence of signal_functions.pyx:222-224, in order: phases[i+1] = (float)(2 pi t[i] (f[i] - f[i+1]) + phases[i]) */
void serial_phases(const float* f, const float* t, long n, float phi, float* ph) {
    if (n <= 0) return;
    ph[0] = phi;
    for (long i = 0; i + 1 < n; i++) ph[i + 1] = (float)(2.0 * M_PI * (double)t[i] * (double)(f[i] - f[i + 1]) + (double)ph[i]);
}
"""


class Libm:
    """libm's sinf / cosf / fmod and the host build of glibc_sincosf.h, through a gcc-built harness (-ffp-contract=off, as the
    restatement is written; numpy's np.sin is not libm)"""

    def __init__(self, td):
        src, so = os.path.join(td, "h.c"), os.path.join(td, "h.so")
        with open(src, "w") as fh:
            fh.write(LIBM_HARNESS % os.path.join(ROOT, "urh_b200", "csrc", "glibc_sincosf.h"))
        subprocess.check_call(["/usr/bin/gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src, "-lm"])
        self.lib = ctypes.CDLL(so)

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    def sincosf(self, y):
        y = np.ascontiguousarray(y, dtype=np.float32)
        sn, cs = np.empty_like(y), np.empty_like(y)
        self.lib.ref(self._p(y), self._p(sn), self._p(cs), ctypes.c_long(len(y)))
        return sn, cs

    def restated(self, y):
        y = np.ascontiguousarray(y, dtype=np.float32)
        sn, cs = np.empty_like(y), np.empty_like(y)
        ok = np.empty(len(y), dtype=np.int32)
        self.lib.restated(self._p(y), self._p(sn), self._p(cs), self._p(ok), ctypes.c_long(len(y)))
        return sn, cs, ok

    def fmod_2pi(self, v):
        v = np.ascontiguousarray(v, dtype=np.float64)
        out = np.empty_like(v)
        self.lib.ref_fmod_2pi(self._p(v), self._p(out), ctypes.c_long(len(v)))
        return out

    def serial_phases(self, f, t, phi):
        f = np.ascontiguousarray(f, dtype=np.float32)
        t = np.ascontiguousarray(t, dtype=np.float32)
        out = np.empty_like(f)
        self.lib.serial_phases(self._p(f), self._p(t), ctypes.c_long(len(f)), ctypes.c_float(phi), self._p(out))
        return out


def near_half_pi_multiples():
    """floats within a few ulps of k * pi / 2 at every magnitude from 1 to 2^127, both signs: the argument reduction's hard cases"""
    ks = np.unique(np.concatenate([np.arange(1, 200), np.round(2.0 ** np.arange(8, 230, 0.37))]))
    x = ks * (np.pi / 2)
    x = x[x < 3.4e38].astype(np.float32)
    steps = np.arange(-4, 5, dtype=np.int64)
    bitsv = (x.view(np.int32).astype(np.int64)[:, None] + steps[None, :]).reshape(-1)
    y = bitsv.astype(np.uint32).view(np.float32)
    y = y[np.isfinite(y)]
    return np.concatenate([y, -y])


def test_host_sincosf_large_arguments():
    """glibc_sincosf.h built for the host equals libm at |x| >= 120 (tests/test_sincosf_restatement.py covers |x| < 120): random
    bit patterns, the top of the float range and floats next to multiples of pi/2"""
    rng = np.random.default_rng(17)
    raw = rng.integers(0, 2 ** 32, 4_000_000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    y = raw[np.isfinite(raw) & (np.abs(raw) >= 120)]
    big = near_half_pi_multiples()
    y = np.concatenate([y, big[np.abs(big) >= 120], np.float32([120.0, -120.0, 3.4028235e38, -3.4028235e38, 2.0 ** 127, 1e30])])
    assert len(y) > 1_500_000
    with tempfile.TemporaryDirectory() as td:
        lm = Libm(td)
        sn, cs, ok = lm.restated(y)
        rs, rc = lm.sincosf(y)
    assert ok.all()
    bad = (sn.view(np.uint32) != rs.view(np.uint32)) | (cs.view(np.uint32) != rc.view(np.uint32))
    # a CPU without FMA/AVX2 selects glibc's SSE2 variant, which may differ in ~2^-29 of the calls
    assert bad.sum() <= 2, (int(bad.sum()), y[bad][:5])


def test_matrix_covers_its_lists():
    """every modulation x dtype pair, bps 1-8, sps, start and sample rate of the lists occurs; some cases take the FSK correction
    fallback (|term| >= 1e15) and have bit counts that are not a multiple of bps"""
    seen = set()
    fallback = ragged = 0
    for bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt in modulator_cases():
        seen.update({("md", mod, np.dtype(dt).name), ("bps", bps), ("sps", sps), ("start", start), ("fs", fs)})
        ragged += len(bits) % bps != 0
        if mod == "FSK":
            t = np.float32(len(bits) // bps * sps + start) / np.float32(fs)
            fallback += 2 * math.pi * float(np.ptp(p)) * float(t) >= 1e15
    assert {("md", m, np.dtype(d).name) for m in MODS for d in DTYPES} <= seen
    assert {("bps", b) for b in range(1, 9)} <= seen
    assert {("sps", s) for s in SPS} | {("start", s) for s in STARTS} | {("fs", f) for f in RATES} <= seen
    assert fallback > 0 and ragged > 0
