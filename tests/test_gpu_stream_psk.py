"""GPU: host PSK captures streamed through a ring of device slots (urh_afp_demod_psk_stream, urh_demod_digitize_psk_stream,
DESIGN.md §4.3 and §4.11) give exactly the resident results.

Each ring chunk continues the Costas loop from the exact state the preceding chunk left on the device, so every sample of the
streamed qad must equal the resident one bit for bit, whatever the chunk size, the ring, the chunk layout of the speculative loop,
the loop bandwidth and where the chunk edges fall (inside a locked burst, in a gap of zeros, on a live spike in a gap, on the first
sample of a burst).  Chunks shorter than 8192 samples (one or three tiles, a short last chunk) run the serial kernel from the
carried state.  Streamed outputs are filled with a NaN sentinel first, so a sample no pass writes cannot match by accident; NaN
outputs compare by position."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits_equal, load_golden
from test_gpu_costas import DTYPES, SCALE, SENTINEL, burst_gap, f32, gpu_psk, layout, psk_burst, spikes

pytestmark = pytest.mark.gpu

TILE = 2048


def _lib():
    from urh_b200 import _lib as L

    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _sentinel(n):
    return np.full(n, SENTINEL, np.uint32).view(np.float32)


def same(got, want, what=""):
    """NaN-aware and bitwise over every sample, sample 0 included; no sentinel left"""
    assert not (got.view(np.uint32) == SENTINEL).any(), ("samples left unwritten", what)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    m = ~np.isnan(want)
    assert bits_equal(got[m], want[m]) == 0, what


def stats(ctx):
    st3, st4 = (C.c_int64 * 3)(), (C.c_int64 * 4)()
    ctx.check(ctx.lib.urh_costas_stats(ctx.handle, st3))
    ctx.check(ctx.lib.urh_costas_stitch_stats(ctx.handle, st4))
    return dict(zip(("fast", "walked", "stepped", "A", "B", "self", "segs"), list(st3) + list(st4)))


def stream_stats(ctx):
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_stream_stats(ctx.handle, st))
    return list(st)


def s_afp(ctx, iq, noise, order, bw, cs, ring):
    n = len(iq)
    out = _sentinel(n)
    ctx.check(ctx.lib.urh_afp_demod_psk_stream(ctx.handle, _ptr(iq), _lib().dtype_code(iq.dtype), n, float(noise), int(order), float(bw),
                                               int(cs), int(ring), _ptr(out)))
    return out


def s_dd(ctx, iq, noise, center, tol, sps, bps, spacing, cs, ring, want_qad=True):
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    k = C.c_int64(0)
    q = _sentinel(len(iq)) if want_qad else None
    ctx.check(ctx.lib.urh_demod_digitize_psk_stream(ctx.handle, _ptr(iq), _lib().dtype_code(iq.dtype), len(iq), float(noise), float(center),
                                                    int(tol), int(sps), int(bps), float(spacing), int(cs), int(ring),
                                                    _ptr(q) if q is not None else None, C.byref(k)))
    return q, _fetch_pulses(ctx, k.value)


def resident(ctx, iq, noise, order, bw=0.1):
    return gpu_psk(ctx, iq, noise, order, bw)[0]


@pytest.fixture
def segs_env(monkeypatch):
    def force(segs):
        if segs is None:
            monkeypatch.delenv("URH_B200_COSTAS_SEGS", raising=False)
        else:
            monkeypatch.setenv("URH_B200_COSTAS_SEGS", str(segs))
    force(None)
    return force


# ---- afp_demod ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", (2, 4, 8))
@pytest.mark.parametrize("dtype", DTYPES)
def test_dtypes_orders_and_layouts(ctx, dtype, order):
    """five dtypes, orders 2, 4 and 8 (run as 4); chunks of one tile, three tiles (the serial kernel per chunk), 2^16 samples and longer
    than the capture (the speculative loop); rings of 2 and 3"""
    n = 150_001
    iq = burst_gap(n, min(order, 4), dtype, seed=order)
    noise = SCALE[dtype][2]
    want = resident(ctx, iq, noise, order)
    for cs, ring in ((TILE, 2), (3 * TILE, 3), (1 << 16, 2), (1 << 18, 3)):
        got = s_afp(ctx, iq, noise, order, 0.1, cs, ring)
        same(got, want, (cs, ring))
        assert stream_stats(ctx)[1] == -(-n // cs)


@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("last", (1, 300, 5000))
def test_short_last_chunk(ctx, order, last):
    """a last chunk of 1, < 512 and < 8192 samples: the serial kernel continued from the state the speculative chunks carried"""
    cs = 1 << 15
    n = 3 * cs + last
    iq = burst_gap(n, order, np.float32, seed=last)
    want = resident(ctx, iq, 0.2, order)
    same(s_afp(ctx, iq, 0.2, order, 0.1, cs, 2), want)


EDGE_CS = 16 * TILE


def edge_capture(order, seed=0):
    """chunk edges of EDGE_CS samples: edge 1 inside a locked burst, edges 2 and 4 inside gaps of zeros, edge 3 on the first sample
    of a burst, edge 5 on a live spike inside a gap (the only sample above the gate near it)"""
    cs = EDGE_CS
    n = 6 * cs + 777
    rng = np.random.default_rng(seed)
    x = psk_burst(n, order, rng)
    x[2 * cs - 5000: 3 * cs] = 0
    x[4 * cs - 3000: 5 * cs + 3000] = 0
    spikes(x, 4 * cs - 2000, 5 * cs + 3000, rng, every=1499)
    x[5 * cs] = np.exp(0.7j)
    return f32(x)


@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("segs", (None, 2, 4, 8, 16))
def test_chunk_edges_layouts_and_bandwidths(ctx, oracle, segs_env, order, segs):
    """edges at the four places above, under every forced chunk layout and loop bandwidths 0.01, 0.1 and 1.0; the natural layout
    at bandwidth 0.1 also against the CPU oracle"""
    iq = edge_capture(order, seed=order)
    segs_env(segs)
    for bw in (0.01, 0.1, 1.0):
        want = resident(ctx, iq, 0.2, order, bw)
        for ring in (2, 3):
            got = s_afp(ctx, iq, 0.2, order, bw, EDGE_CS, ring)
            same(got, want, (bw, ring))
        if segs is None and bw == 0.1:
            ref = oracle.afp_demod(iq, 0.2, "PSK", order, bw)
            assert got[0] == 0 and bits_equal(got[1:], ref[1:]) == 0


# ---- demod_digitize -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bps", (1, 2))
@pytest.mark.parametrize("tol", (0, 5, 40_000))
def test_demod_digitize(ctx, sf, tol, bps):
    """qad and rows equal urh_demod_digitize for PSK (Costas loop of order 2^bps, then grab_pulse_lens); tolerance 0, 5 and longer
    than a chunk; with and without the host qad"""
    n = 200_003
    iq = burst_gap(n, 1 << bps, np.float32, seed=bps)
    spacing = 0.5 if bps == 2 else 0.1
    q0, r0 = sf.demod_digitize(iq, 0.2, "PSK", 0.0, tol, 300, bits_per_symbol=bps, center_spacing=spacing)
    for cs, ring in ((1 << 15, 2), (3 * TILE, 3)):
        q1, r1 = s_dd(ctx, iq, 0.2, 0.0, tol, 300, bps, spacing, cs, ring)
        same(q1, q0, (cs, ring))
        assert np.array_equal(r1, r0), (cs, ring)
        _, r2 = s_dd(ctx, iq, 0.2, 0.0, tol, 300, bps, spacing, cs, ring, want_qad=False)
        assert np.array_equal(r2, r0), (cs, ring)


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


# ---- diagnostics ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("segs", (4, 16))
def test_summed_diagnostics(ctx, segs_env, order, segs):
    """after a streamed call the counters are sums over the ring chunks: O(1) + walked = sum of (chunks - 1), the stitch resolved
    sum of (super-chunks - 1), and most chunks still resolve in O(1) (the stream did not fall back to serial speed)"""
    segs_env(segs)
    n, cs = 1_000_003, 1 << 18
    iq = burst_gap(n, order, np.float32, seed=7)
    want = resident(ctx, iq, 0.2, order)
    same(s_afp(ctx, iq, 0.2, order, 0.1, cs, 2), want)
    st = stats(ctx)
    lens = [min(cs, n - s) for s in range(0, n, cs)]
    chunks = [layout(m, segs)[0] for m in lens]
    supers = [layout(m, segs)[1] for m in lens]
    assert st["segs"] == segs, st
    assert st["fast"] + st["walked"] == sum(c - 1 for c in chunks), (st, chunks)
    assert st["A"] + st["B"] + st["self"] == sum(s - 1 for s in supers), (st, supers)
    assert st["fast"] >= 0.7 * sum(chunks), (st, chunks)
    assert 0 < st["stepped"] <= n


# ---- device memory --------------------------------------------------------------------------------------------------------------
def _psk_calls(ctx, iq, tol, cs, ring):
    L = _lib()
    from urh_b200.cythonext.signal_functions import psk_entry

    noise = SCALE[np.int16][2]
    return [
        (L.STREAM_AFP_DEMOD | psk_entry(4), lambda: (s_afp(ctx, iq, noise, 4, 0.1, cs, ring), None)),
        (L.STREAM_DEMOD_DIGITIZE | L.STREAM_QAD_OUT | psk_entry(2), lambda: s_dd(ctx, iq, noise, 0.0, tol, 300, 1, 0.1, cs, ring)),
        (L.STREAM_DEMOD_DIGITIZE | psk_entry(4), lambda: s_dd(ctx, iq, noise, 0.0, tol, 300, 2, 0.5, cs, ring, want_qad=False)),
    ]


@pytest.mark.parametrize("tol", (0, 5))
def test_device_memory_within_footprint(sf, ctx, tol):
    """device memory in use during a streamed PSK call (urh_mem_get_info before, the low point urh_stream_stats saw inside) stays
    within urh_stream_footprint for the PSK entry"""
    n, cs, ring = (1 << 22) + 5, 1 << 18, 3
    iq = burst_gap(n, 4, np.int16, seed=8)
    ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 1))
    try:
        for entry, call in _psk_calls(ctx, iq, tol, cs, ring):
            ctx.sync()
            free, total = C.c_size_t(0), C.c_size_t(0)
            ctx.check(ctx.lib.urh_mem_get_info(ctx.handle, C.byref(free), C.byref(total)))
            _, rows = call()
            st = stream_stats(ctx)
            assert st[1] == (n + cs - 1) // cs and st[0] > 0
            used = free.value - st[0]
            assert used <= sf.stream_footprint(n, np.int16, tol, entry, cs, ring, 0 if rows is None else len(rows)), (entry, used)
    finally:
        ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 0))


def test_scratch_does_not_grow_with_n(ctx):
    """the Costas loop's candidates, checkpoints and chain tables are sized per chunk: the most scratch-arena bytes live at once are
    the same for a capture 4x longer"""
    cs, ring = 1 << 18, 2
    peaks = {}
    base = burst_gap((1 << 22) + 5, 4, np.int16, seed=8)
    for n in ((1 << 22) + 5, (1 << 24) + 5):
        iq = np.ascontiguousarray(np.resize(base, (n, 2)))
        for entry, call in _psk_calls(ctx, iq, 5, cs, ring):
            call()
            peaks.setdefault(entry, []).append(stream_stats(ctx)[2])
    for entry, (small, big) in peaks.items():
        assert big == small > 0, (entry, small, big)


# ---- the public functions -------------------------------------------------------------------------------------------------------
def test_shims_choose_stream(sf, ctx, monkeypatch, tmp_path):
    """a low $URH_B200_DEVICE_BUDGET makes afp_demod and demod_digitize stream a host PSK capture (several chunks), with the resident
    results for pinned, pageable and memory-mapped sources; with the default budget a small capture stays resident"""
    from urh_b200.device import PinnedArray

    L = _lib()
    n = 3 * (1 << 16) + 77
    iq = burst_gap(n, 4, np.float32, seed=4)
    assert not sf.use_stream(n, iq.dtype, 5, L.STREAM_AFP_DEMOD | sf.psk_entry(4), sf.device_budget(ctx))
    # a streamed call of known chunk count first: the shims' resident calls below must leave urh_stream_stats as it is
    s_afp(ctx, iq, 0.2, 4, 0.05, 5 * TILE, 2)
    marker = stream_stats(ctx)[1]
    assert marker == -(-n // (5 * TILE))
    a0 = sf.afp_demod(iq, 0.2, "PSK", 4, 0.05)
    d0 = sf.demod_digitize(iq, 0.2, "PSK", 0.0, 5, 300, bits_per_symbol=2, center_spacing=0.5)
    assert stream_stats(ctx)[1] == marker, "a capture that fits the default budget was streamed"
    pinned = PinnedArray(iq.shape, iq.dtype)
    pinned.array[:] = iq
    mm = np.memmap(tmp_path / "cap.f32", dtype=np.float32, mode="w+", shape=iq.shape)
    mm[:] = iq
    mm.flush()
    monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(1 << 20))
    monkeypatch.setattr(sf, "PSK_STREAM_CHUNK", 1 << 16)
    assert sf.use_stream(n, iq.dtype, 5, L.STREAM_DEMOD_DIGITIZE | sf.psk_entry(4), sf.device_budget(ctx))
    for src in (iq, pinned.array, np.memmap(tmp_path / "cap.f32", dtype=np.float32, mode="r", shape=iq.shape)):
        same(sf.afp_demod(src, 0.2, "PSK", 4, 0.05), a0)
        assert stream_stats(ctx)[1] == 4
        q, r = sf.demod_digitize(src, 0.2, "PSK", 0.0, 5, 300, bits_per_symbol=2, center_spacing=0.5)
        assert stream_stats(ctx)[1] == 4
        same(q, d0[0])
        assert np.array_equal(r, d0[1])
    pinned.free()


def test_signal_and_protocol_analyzer_stream(sf, monkeypatch):
    """Signal.qad and ProtocolAnalyzer.get_protocol_from_signal on a PSK capture under a budget of 64 KiB: demodulation and
    digitizer stream from the host, nothing stays on the device, the messages are the resident run's and the golden bits"""
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.ProtocolAnalyzer import ProtocolAnalyzer
    from urh_b200.signalprocessing.Signal import Signal

    g = load_golden("capture_psk_gen_noisy")
    m = g["meta"]

    def run():
        s = Signal("", "psk")
        s.iq_array = IQArray(g["iq"])
        s.noise_threshold = float(g["noise"])
        s.modulation_type = m["mod"]
        s.samples_per_symbol = m["sps"]
        s.center = m["center"]
        s.tolerance = m["tol"]
        s.bits_per_symbol = m["bps"]
        s.center_spacing = m["spacing"]
        pa = ProtocolAnalyzer(s)
        pa.get_protocol_from_signal()
        return s, pa

    s0, pa0 = run()
    assert s0._qad_dev is not None
    monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(1 << 16))
    monkeypatch.setattr(sf, "PSK_STREAM_CHUNK", TILE)
    s1, pa1 = run()
    assert s1._qad_dev is None and s1.iq_array._device is None and s1.qad_device is None
    assert bits_equal(s1.qad, s0.qad) == 0
    assert pa1.plain_bits_str == pa0.plain_bits_str == m["bits"]


def test_default_chunk_long_capture(sf, ctx):
    """2^28 float32 samples at order 4 through the default PSK chunk equal the resident result as a whole"""
    n = 1 << 28
    base = burst_gap(1 << 22, 4, np.float32, seed=3, period=300_000, gap=50_000)
    iq = np.resize(base, (n, 2))
    want = resident(ctx, iq, 0.2, 4)
    got = s_afp(ctx, iq, 0.2, 4, 0.1, sf.PSK_STREAM_CHUNK, 2)
    same(got, want)
    assert stream_stats(ctx)[1] == -(-n // sf.PSK_STREAM_CHUNK)
