"""GPU: the PSK demodulator (Costas loop) against the serial recurrence of the oracle (== the reference's costa_demod), bit for bit.

Paths: captures shorter than 8192 samples run the serial kernel (costas.cu, k_costas); longer ones the speculative chunk-parallel
loop (costas_spec.cu).  Each speculative case also asserts the path it took, through urh_costas_stats ({O(1) chunks, walked chunks,
stepped samples}) and urh_costas_stitch_stats ({super-chunks adopted from family A, from family B, chained by the stitch warp,
segs}): the speculation is exact by construction, so most of its bugs would make it slower, not wrong.  $URH_B200_COSTAS_SEGS
forces every chunk layout (2, 4, 8, 16 segments of 256 samples per chunk) on captures of any length.

The output buffer is filled with a NaN sentinel before every call, so a sample that no pass writes cannot pass by accident."""
import ctypes as C
import time

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

DTYPES = (np.int8, np.uint8, np.int16, np.uint16, np.float32)
SEGS = (2, 4, 8, 16)
SENTINEL = np.uint32(0x7FBADBAD)   # a NaN payload neither kernel produces
SEG = 256   # samples per segment (costas_spec.cu: CS_SEG)


def synth_psk(n, order, sps=300, sigma=0.05, seed=0, gap_period=600000, gap_len=100000, dtype=np.float32):
    rng = np.random.default_rng(seed)
    nsym = n // sps + 1
    sym = rng.integers(0, order, nsym)
    ph = 2 * np.pi * 0.025 * np.arange(n) + np.repeat(2 * np.pi * sym / order + (np.pi / 4 if order == 4 else 0), sps)[:n]
    on = (np.arange(n) % gap_period) < (gap_period - gap_len)
    x = on * np.exp(1j * ph) + sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    iq = np.empty((n, 2), np.float32)
    iq[:, 0] = x.real
    iq[:, 1] = x.imag
    if dtype == np.int8:
        return np.clip(iq * 100, -128, 127).astype(np.int8)
    return iq


# scale of a unit-amplitude sample, offset of zero and a noise gate that passes the bursts and stops the gaps, per dtype.  The
# gate compares the RAW values (pyx:293), so the unsigned captures get gaps of exact zeros (a centred gap would not be gated).
SCALE = {np.int8: (100, 0, 20.0), np.uint8: (100, 128, 20.0), np.int16: (20000, 0, 4000.0), np.uint16: (20000, 32768, 4000.0),
         np.float32: (1, 0, 0.2)}


def to_dtype(x, on, dtype):
    """complex capture -> IQ samples of `dtype`; the unsigned kinds get exact zeros where `on` is False"""
    iq = np.stack([x.real, x.imag], axis=1)
    if dtype == np.float32:
        return np.ascontiguousarray(iq, dtype=np.float32)
    scale, zero, _ = SCALE[dtype]
    info = np.iinfo(dtype)
    out = np.clip(np.round(iq * scale + zero), info.min, info.max).astype(dtype)
    if zero:
        out[~on] = 0
    return out


def burst_gap(n, order, dtype=np.float32, seed=0, period=30000, gap=9000, sigma=0.05):
    """PSK bursts (300 samples per symbol, a carrier offset of 0.025 cycles per sample) with noise-only gaps of `gap` samples
    every `period` samples"""
    rng = np.random.default_rng(seed)
    sym = rng.integers(0, order, n // 300 + 1)
    ph = 2 * np.pi * 0.025 * np.arange(n) + np.repeat(2 * np.pi * sym / order + (np.pi / 4 if order == 4 else 0), 300)[:n]
    on = (np.arange(n) % period) < (period - gap)
    x = on * np.exp(1j * ph) + sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return to_dtype(x, on, dtype)


def layout(n, segs):
    """(chunks, super-chunks) of the speculative path (costas_spec.cu: cs_speculate)"""
    chunk = segs * SEG
    nchunks = -(-n // chunk)
    sup = max(64, -(-131072 // chunk))
    return nchunks, -(-nchunks // sup)


def default_segs(ctx, n, order):
    sm = ctx.device_info()["sm_count"]
    segs = 16
    while segs > 2 and (n // (segs * SEG)) * min(order, 4) < sm * 1024:
        segs >>= 1
    return segs


def gpu_psk(ctx, iq, noise, order, bw=0.1):
    """urh_afp_demod(PSK) into a sentinel-filled buffer -> (result, {fast, walked, stepped, A, B, self, segs})"""
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device

    n = len(iq)
    d_iq = to_device(np.ascontiguousarray(iq), ctx)
    out = DeviceArray(ctx, (n,), np.float32)
    out.set(np.full(n, SENTINEL, np.uint32).view(np.float32))
    ctx.check(ctx.lib.urh_afp_demod(ctx.handle, C.c_void_p(d_iq.ptr), _lib.dtype_code(iq.dtype), n, float(noise), _lib.MOD_PSK,
                                    int(order), float(bw), C.c_void_p(out.ptr)))
    q = out.get()
    st3, st4 = (C.c_int64 * 3)(), (C.c_int64 * 4)()
    ctx.check(ctx.lib.urh_costas_stats(ctx.handle, st3))
    ctx.check(ctx.lib.urh_costas_stitch_stats(ctx.handle, st4))
    stats = dict(zip(("fast", "walked", "stepped", "A", "B", "self", "segs"), list(st3) + list(st4)))
    assert stats["self"] == ctx.lib.urh_costas_last_redone(ctx.handle)
    assert not (q.view(np.uint32) == SENTINEL).any(), "samples left unwritten"
    return q, stats


def assert_exact(got, want, what=""):
    assert bits_equal(got[1:], want[1:]) == 0, what
    assert got[0] == 0 and want[0] == 0


def assert_path(stats, n, order, segs=None, what=""):
    """the counters are consistent with the path the length selects: the serial kernel below 8192 samples"""
    if n < 8192 or min(order, 4) not in (2, 4):
        assert stats == dict(fast=0, walked=0, stepped=0, A=0, B=0, self=0, segs=0), (what, stats)
        return
    if segs is not None:
        assert stats["segs"] == segs, (what, stats)
    nchunks, nsuper = layout(n, stats["segs"])
    # chunk 0 and super-chunk 0 of the capture have one run only: they are not counted
    assert stats["fast"] + stats["walked"] == nchunks - 1, (what, stats)
    assert stats["A"] + stats["B"] + stats["self"] == nsuper - 1, (what, stats)
    assert stats["stepped"] <= n


def run(ctx, oracle, iq, noise, order, bw=0.1, segs=None, what=""):
    got, stats = gpu_psk(ctx, iq, noise, order, bw)
    assert_exact(got, oracle.afp_demod(iq, noise, "PSK", order, bw), what)
    assert_path(stats, len(iq), order, segs, what)
    return stats


@pytest.fixture
def force_segs(monkeypatch):
    def force(segs):
        if segs is None:
            monkeypatch.delenv("URH_B200_COSTAS_SEGS", raising=False)
        else:
            monkeypatch.setenv("URH_B200_COSTAS_SEGS", str(segs))   # read by getenv() on every call (costas_spec.cu)
    force(None)
    return force


# ---- the existing end-to-end cases (signal_functions.afp_demod) ----------------------------------------------------------------

@pytest.mark.parametrize("order,dtype,noise", [(2, np.float32, 0.2), (4, np.float32, 0.2), (2, np.int8, 20.0), (2, np.float32, 0.0)])
def test_speculative_costas_bit_exact(oracle, ctx, force_segs, order, dtype, noise):
    from urh_b200.cythonext import signal_functions as sf

    n = 1_500_000
    iq = synth_psk(n, order, seed=order, dtype=dtype)
    t0 = time.time()
    q = sf.afp_demod(iq, noise, "PSK", order)
    t_gpu = time.time() - t0
    ref = oracle.afp_demod(iq, noise, "PSK", order)
    assert bits_equal(q[1:], ref[1:]) == 0
    st = (C.c_int64 * 3)()
    ctx.lib.urh_costas_stats(ctx.handle, st)
    # the speculation must carry almost all chunks (otherwise the kernel silently degrades to the serial loop)
    assert st[0] >= 0.7 * (n // 4096), list(st)
    print("costas order", order, "gpu %.3fs" % t_gpu, "fast/slow/stepped", list(st))


def test_speculative_costas_edge_sizes(oracle, force_segs):
    from urh_b200.cythonext import signal_functions as sf

    for n in (4 * 4096, 4 * 4096 + 1, 5 * 4096 - 1, 100_003):
        iq = synth_psk(n, 2, seed=n, gap_period=30000, gap_len=9000)
        assert bits_equal(sf.afp_demod(iq, 0.2, "PSK", 2)[1:], oracle.afp_demod(iq, 0.2, "PSK", 2)[1:]) == 0, n
        iq[:] = 0
        assert bits_equal(sf.afp_demod(iq, 0.2, "PSK", 2)[1:], oracle.afp_demod(iq, 0.2, "PSK", 2)[1:]) == 0


# ---- (a) sizes around every switch, every dtype and loop order -----------------------------------------------------------------

# 3 .. 4097: the COSTAS_CHUNK = 2048 staging of k_costas; 8191 | 8192: the serial / speculative switch; 300 001 leaves the last
# chunk, the last 32-chunk prefetch group of cs_chain and the last super-chunk partial in every layout (and 225 samples in the
# last segment, a partial k_cs_fix segment); 131 073: a last super-chunk of one chunk of one sample at segs = 2 and 4
SIZES = (3, 4, 2047, 2048, 2049, 4097, 8191, 8192, 8193, 16383, 16384, 131_073, 300_001)


def sizes_capture(n, order, dtype):
    period = min(30000, max(n // 4, 64))
    return burst_gap(n, order, dtype, seed=n + order, period=period, gap=period * 3 // 10)


@pytest.mark.parametrize("order", (2, 4, 8))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_sizes_around_every_switch(oracle, ctx, force_segs, dtype, order):
    noise = SCALE[dtype][2]
    for n in SIZES:
        iq = sizes_capture(n, order, dtype)
        run(ctx, oracle, iq, noise, order, segs=default_segs(ctx, n, order) if n >= 8192 else None, what=n)


# ---- (b) every chunk layout --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("segs", SEGS)
@pytest.mark.parametrize("order", (2, 4, 8))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_every_chunk_layout(oracle, ctx, force_segs, dtype, order, segs):
    force_segs(segs)
    noise = SCALE[dtype][2]
    for n in [s for s in SIZES if s >= 8192]:
        run(ctx, oracle, sizes_capture(n, order, dtype), noise, order, segs=segs, what=n)
    # the throughput guard on an ordinary burst-and-gap capture (bursts of 21 000 samples, gaps of 9 000)
    n = 1_000_003
    st = run(ctx, oracle, burst_gap(n, order, dtype, seed=segs), noise, order, segs=segs)
    # (a uint16 capture scaled by 65535 has a third of the amplitude, and the order-2 loop then merges more slowly than the
    # 1024-sample warm-up: exact, but not fast)
    if order in (2, 4) and not (dtype == np.uint16 and order == 2):
        assert st["fast"] >= 0.7 * layout(n, segs)[0], st


# ---- (c) constructed inputs that force each branch ------------------------------------------------------------------------------

S16 = 64 * 16 * SEG   # the longest super-chunk (segs = 16); every other layout has 131 072-sample super-chunks


def psk_burst(n, order, rng, sigma=0.05):
    sym = rng.integers(0, order, n // 300 + 1)
    ph = 2 * np.pi * 0.025 * np.arange(n) + np.repeat(2 * np.pi * sym / order, 300)[:n] + rng.uniform(0, 2 * np.pi)
    return np.exp(1j * ph) + sigma * (rng.standard_normal(n) + 1j * rng.standard_normal(n))


def spikes(x, lo, hi, rng, every=997):
    """isolated unit samples of random phase in [lo, hi): above the gate, too sparse for any two trajectories to merge"""
    idx = np.arange(lo, hi, every)
    x[idx] = np.exp(2j * np.pi * rng.random(len(idx)))
    return x


def f32(x):
    return np.ascontiguousarray(np.stack([x.real, x.imag], axis=1), dtype=np.float32)


@pytest.mark.parametrize("segs", SEGS)
@pytest.mark.parametrize("order", (2, 4))
def test_family_a_locked_burst(oracle, ctx, force_segs, order, segs):
    """one locked burst over every super-chunk boundary: every super-chunk is adopted from family A"""
    force_segs(segs)
    n = 3 * S16 + 1000
    st = run(ctx, oracle, f32(psk_burst(n, order, np.random.default_rng(order))), 0.2, order, segs=segs)
    assert st["A"] == layout(n, segs)[1] - 1 and st["B"] == 0 and st["self"] == 0, st
    assert st["fast"] >= 0.9 * layout(n, segs)[0], st


@pytest.mark.parametrize("segs", SEGS)
@pytest.mark.parametrize("order", (2, 4))
def test_family_b_gap_of_zeros(oracle, ctx, force_segs, order, segs):
    """a gap of exact zeros over a super-chunk boundary after a locked burst: the loop state is frozen there, no warm-up
    reproduces it, family B (the end state of the preceding chain) does"""
    force_segs(segs)
    n = 4 * S16
    rng = np.random.default_rng(10 + order)
    x = psk_burst(n, order, rng)
    x[int(1.55 * S16): int(2.6 * S16)] = 0
    st = run(ctx, oracle, f32(x), 0.2, order, segs=segs)
    assert st["B"] > 0 and st["A"] > 0 and st["self"] == 0, st


@pytest.mark.parametrize("segs", SEGS)
@pytest.mark.parametrize("order", (2, 4))
def test_stitch_chains_itself_in_a_creeping_gap(oracle, ctx, force_segs, order, segs):
    """a gap with isolated spikes over whole super-chunks: the frozen state creeps, neither family starts in it, the stitch
    warp runs the chain itself"""
    force_segs(segs)
    n = int(4.5 * S16)
    rng = np.random.default_rng(20 + order)
    x = psk_burst(n, order, rng)
    lo, hi = int(1.2 * S16), int(3.5 * S16)
    x[lo:hi] = 0
    spikes(x, lo + 500, hi, rng)
    st = run(ctx, oracle, f32(x), 0.2, order, segs=segs)
    assert st["A"] > 0 and st["B"] > 0, st
    if order == 2:
        assert st["self"] > 0, st
    else:   # the sign detector of order 4 can pull a candidate onto the true state over 262 144 samples of spikes (segs 16)
        assert st["B"] + st["self"] >= 2, st


@pytest.mark.parametrize("segs", SEGS)
@pytest.mark.parametrize("order", (2, 4))
def test_walked_chunks_with_bursts_starting_mid_chunk(oracle, ctx, force_segs, order, segs):
    """bursts starting at odd offsets, at loop bandwidth 0.01 (slow merges): merges land mid-chunk, on the last segment, or
    not within the chunk; the stepped segments hold gated samples in front of the burst (k_cs_fix)"""
    force_segs(segs)
    rng = np.random.default_rng(30 + order)
    n = 700_001
    x = np.zeros(n, np.complex128)
    pos = 1000
    while pos < n:
        length = int(rng.integers(3000, 40000))
        x[pos: pos + length] = psk_burst(min(length, n - pos), order, rng)
        pos += length + int(rng.integers(200, 9000)) + int(rng.integers(0, 256))
    for bw in (0.01, 0.1):
        st = run(ctx, oracle, f32(x), 0.2, order, bw=bw, segs=segs, what=bw)
        assert st["walked"] > 0 and st["stepped"] > 0, st


@pytest.mark.parametrize("segs", SEGS)
def test_pure_noise_degrades_to_serial_speed(oracle, ctx, force_segs, segs):
    """complex noise with gate 0 at bandwidth 1.0: trajectories rarely merge, most chunks are walked; still exact"""
    force_segs(segs)
    rng = np.random.default_rng(40)
    n = 200_003
    iq = f32(rng.standard_normal(n) + 1j * rng.standard_normal(n))
    for order in (2, 4):
        st = run(ctx, oracle, iq, 0.0, order, bw=1.0, segs=segs, what=order)
        assert st["walked"] >= 0.75 * layout(n, segs)[0], st


@pytest.mark.parametrize("segs", SEGS)
def test_all_noise_chunks_and_segments(oracle, ctx, force_segs, segs):
    """short bursts between gaps of zeros: whole chunks of noise (the ccnt == 0 shortcut) and all-noise segments inside walked
    chunks (cnt == 0)"""
    force_segs(segs)
    rng = np.random.default_rng(50)
    n = 600_000
    x = np.zeros(n, np.complex128)
    pos = 10
    while pos < n:
        length = int(rng.integers(50, 400))
        x[pos: pos + length] = psk_burst(min(length, n - pos), 2, rng)
        pos += length + int(rng.choice([300, 700, 5000, 20000]))
    for order in (2, 4):
        run(ctx, oracle, f32(x), 0.2, order, segs=segs, what=order)
        run(ctx, oracle, to_dtype(x, np.abs(x) > 0, np.int16), 4000.0, order, segs=segs, what=order)


# ---- (d) loop bandwidth ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bw", (0.01, 0.05, 0.1, 0.3, 1.0))
@pytest.mark.parametrize("order", (2, 4))
def test_loop_bandwidth_sweep(oracle, ctx, force_segs, order, bw):
    n = 1_000_003
    run(ctx, oracle, burst_gap(n, order, np.float32, seed=60 + order), 0.2, order, bw=bw)


def test_signal_passes_order_and_bandwidth(oracle, ctx, force_segs):
    """Signal with bits_per_symbol = 3 (mod_order 8 -> loop order 4) and a non-default costas_loop_bandwidth"""
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.Signal import Signal

    iq = burst_gap(400_000, 8, np.float32, seed=70)
    s = Signal("", "psk8")
    s.iq_array = IQArray(iq)
    s.noise_threshold = 0.2
    s.modulation_type = "PSK"
    s.bits_per_symbol = 3
    s.costas_loop_bandwidth = 0.3
    want = oracle.afp_demod(iq, 0.2, "PSK", 8, 0.3)
    assert bits_equal(s.qad[1:], want[1:]) == 0
    assert bits_equal(want[1:], oracle.afp_demod(iq, 0.2, "PSK", 8, 0.1)[1:]) > 0   # the bandwidth reached the loop


# ---- (e) edges of the arithmetic ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("segs", (None, 2, 16))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_samples_exactly_on_the_gate(oracle, ctx, force_segs, dtype, segs):
    """re^2 + im^2 == noise^2 is noise, one step above is not: (3, 4) is noise and (3, 5) is not, with noise 5"""
    force_segs(segs)
    rng = np.random.default_rng(80)
    for n in (5000, 100_003):
        on_gate, above, noise = (3, 4), (3, 5), 5.0
        pick = rng.random(n)
        iq = np.where((pick < 0.5)[:, None], np.array(on_gate), np.array(above))
        flip = rng.random((n, 2)) < 0.5
        if not np.issubdtype(dtype, np.unsignedinteger):
            iq = np.where(flip, -iq, iq)   # the sign does not move a sample across the gate, it moves the loop
        iq = np.ascontiguousarray(iq, dtype=dtype)
        assert (oracle.afp_demod(iq, noise, "PSK", 2)[1:] == -4.0).sum() == (pick[1:] < 0.5).sum()
        for order in (2, 4):
            run(ctx, oracle, iq, noise, order, what=(n, order))


def nan_aware_equal(got, want):
    """NaN at the same positions (its payload may differ between the GPU and x86), every other word bitwise equal"""
    g, w = got[1:], want[1:]
    assert np.array_equal(np.isnan(g), np.isnan(w))
    m = ~np.isnan(w)
    assert bits_equal(g[m], w[m]) == 0


@pytest.mark.parametrize("segs", (None, 2, 16))
@pytest.mark.parametrize("order", (2, 4))
def test_huge_and_infinite_samples(oracle, ctx, force_segs, order, segs):
    """float32 samples of +-1e30 and +-inf in the real part: the error clamp keeps the order-2 loop state finite, bitwise bar.
    inf in the imaginary part reaches the Annex G recovery of the complex product: infinite, not NaN"""
    force_segs(segs)
    for n in (6000, 300_001):
        base = burst_gap(n, order, np.float32, seed=90, period=20000, gap=5000)
        for val in ((1e30, -1e30), (-1e30, 1e30), (np.inf, 0.0), (-np.inf, 0.0), (0.3, np.inf), (-0.3, -np.inf), (np.inf, np.inf)):
            iq = base.copy()
            iq[n // 3] = val
            iq[n // 3 + 7] = val
            iq[n - 2] = val
            got, stats = gpu_psk(ctx, iq, 0.2, order)
            want = oracle.afp_demod(iq, 0.2, "PSK", order)
            nan_aware_equal(got, want)
            assert_path(stats, n, order, segs)
            if order == 2:
                assert not np.isnan(want).any(), val   # the loop state stays finite
                assert_exact(got, want, val)


@pytest.mark.parametrize("segs", (None, 2, 16))
@pytest.mark.parametrize("order", (2, 4))
def test_nan_samples(oracle, ctx, force_segs, order, segs):
    """a NaN sample makes the loop state NaN from then on (every later live sample is NaN)"""
    force_segs(segs)
    for n in (6000, 300_001):
        base = burst_gap(n, order, np.float32, seed=95, period=20000, gap=5000)
        for val in ((np.nan, 0.5), (0.5, np.nan)):
            iq = base.copy()
            iq[n // 2] = val
            got, stats = gpu_psk(ctx, iq, 0.2, order)
            want = oracle.afp_demod(iq, 0.2, "PSK", order)
            nan_aware_equal(got, want)
            assert np.isnan(want[n // 2:][want[n // 2:] != -4.0]).all()
            assert_path(stats, n, order, segs)


# ---- (f) the natural layout of a long capture -------------------------------------------------------------------------------------

def test_natural_layout_of_a_long_capture(oracle, ctx, force_segs):
    """2^28 float32 samples, order 4, no override: on an H100 (132 SMs) this selects segs = 16"""
    n = 1 << 28
    block = burst_gap(1 << 22, 4, np.float32, seed=100, period=600000, gap=100000)
    iq = np.tile(block, (n >> 22, 1))
    got, stats = gpu_psk(ctx, iq, 0.2, 4)
    want = oracle.afp_demod(iq, 0.2, "PSK", 4)
    assert_exact(got, want)
    assert_path(stats, n, 4, default_segs(ctx, n, 4))
    if ctx.device_info()["sm_count"] == 132:
        assert stats["segs"] == 16
    assert stats["fast"] >= 0.7 * layout(n, stats["segs"])[0], stats
