"""GPU: host captures streamed through a ring of device slots (urh_*_stream, DESIGN.md §4.11) give exactly the resident results.

Every case compares the streamed call with the resident one word for word: qad (bits_equal), pulse rows, center, center_state and
urh_center_certify_stats.  Chunks of one tile and of odd tile counts, captures shorter than a chunk and not a multiple of a tile,
tolerances 0, 5 and longer than a chunk (runs that span several chunks), rings of 2 and 3 slots."""
import ctypes as C

import numpy as np
import pytest

from conftest import CAPTURES, bits_equal, load_golden, synth_fsk

pytestmark = pytest.mark.gpu

TILE = 2048
DTYPES = [np.float32, np.int16, np.uint16, np.int8, np.uint8]
NOISE = {np.float32: 0.05, np.int16: 1000.0, np.uint16: 1000.0, np.int8: 5.0, np.uint8: 5.0}


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _lib():
    from urh_b200 import _lib as L

    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _capture(n, dtype, mod, seed=11):
    iq = synth_fsk(n, seed=seed, gap_every=9_000, dtype=dtype)
    if mod == "ASK":
        env = np.repeat(np.random.default_rng(seed + 1).integers(0, 2, n // 100 + 1), 100)[:n] * 0.8 + 0.2
        iq = (iq.astype(np.float32) * env[:, None]).astype(dtype)
    return np.ascontiguousarray(iq)


def _code(mod):
    L = _lib()
    return L.MOD_ASK if mod == "ASK" else L.MOD_FSK


# ---- the streamed entry points, called with an explicit chunk size and ring ----------------------------------------------------
def s_afp(ctx, iq, noise, mod, cs, ring):
    L = _lib()
    out = np.empty(len(iq), np.float32)
    ctx.check(ctx.lib.urh_afp_demod_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), len(iq), float(noise), _code(mod), cs, ring, _ptr(out)))
    return out


def s_grab(ctx, qad, center, tol, mod, sps, bps, cs, ring, spacing=0.1):
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    k = C.c_int64(0)
    ctx.check(ctx.lib.urh_grab_pulse_lens_stream(ctx.handle, _ptr(qad), 0, len(qad), float(center), tol, _code(mod), sps, bps, spacing, cs, ring,
                                                 C.byref(k)))
    return _fetch_pulses(ctx, k.value)


def s_dd(ctx, iq, noise, mod, center, tol, sps, cs, ring, want_qad=True):
    from urh_b200.cythonext.signal_functions import _fetch_pulses

    L = _lib()
    k = C.c_int64(0)
    q = np.empty(len(iq), np.float32) if want_qad else None
    ctx.check(ctx.lib.urh_demod_digitize_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), len(iq), float(noise), _code(mod), float(center),
                                                tol, sps, 1, 0.1, cs, ring, _ptr(q) if q is not None else None, C.byref(k)))
    return q, _fetch_pulses(ctx, k.value)


def _cert(ctx):
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_center_certify_stats(ctx.handle, st))
    return list(st)


def s_center(ctx, iq, noise, mod, tol, sps, cs, ring, max_size=None):
    from urh_b200.cythonext.signal_functions import _fetch_pulses
    from urh_b200.device import DeviceArray

    L = _lib()
    n = len(iq)
    d_qad = DeviceArray(ctx, (n,), np.float32)
    ctx.check(ctx.lib.urh_memset(ctx.handle, C.c_void_p(d_qad.ptr), 0xFF, 4 * n))   # NaN: a sample the call misses cannot match
    h_qad = np.full(n, np.nan, np.float32)
    center, state, kept, k = C.c_double(0.0), C.c_int(0), C.c_int64(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_demod_center_digitize_stream(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), n, float(noise), _code(mod), tol, sps,
                                                       -1 if max_size is None else max_size, cs, ring, C.c_void_p(d_qad.ptr), _ptr(h_qad),
                                                       C.byref(center), C.byref(state), C.byref(kept), C.byref(k)))
    rows = _fetch_pulses(ctx, k.value) if state.value == 1 else np.zeros((0, 2), np.int64)
    assert bits_equal(d_qad.get(), h_qad) == 0   # the host mirror is the resident qad
    return state.value, (center.value if state.value == 1 else None), rows, h_qad, _cert(ctx)


def r_center(ctx, iq, noise, mod, tol, sps, max_size=None):
    """the resident one-call step (urh_demod_center_digitize_host with the whole capture on the device)"""
    from urh_b200.cythonext.signal_functions import _fetch_pulses
    from urh_b200.device import DeviceArray

    L = _lib()
    n = len(iq)
    d_iq = DeviceArray(ctx, iq.shape, iq.dtype)
    d_qad = DeviceArray(ctx, (n,), np.float32)
    center, state, k = C.c_double(0.0), C.c_int(0), C.c_int64(0)
    ctx.check(ctx.lib.urh_demod_center_digitize_host(ctx.handle, _ptr(iq), L.dtype_code(iq.dtype), n, float(noise), _code(mod), tol, sps,
                                                     -1 if max_size is None else max_size, 0, C.c_void_p(d_iq.ptr), C.c_void_p(d_qad.ptr),
                                                     C.byref(center), C.byref(state), C.byref(k)))
    rows = _fetch_pulses(ctx, k.value) if state.value == 1 else np.zeros((0, 2), np.int64)
    return state.value, (center.value if state.value == 1 else None), rows, d_qad.get(), _cert(ctx)


def _check_all(sf, ctx, iq, noise, mod, tol, cs, ring, sps=100, center=None, max_size=None):
    """every streamed entry against its resident twin"""
    qad = sf.afp_demod(iq, noise, mod, 2)
    assert bits_equal(s_afp(ctx, iq, noise, mod, cs, ring), qad) == 0
    rs = r_center(ctx, iq, noise, mod, tol, sps, max_size)
    ss = s_center(ctx, iq, noise, mod, tol, sps, cs, ring, max_size)
    assert ss[0] == rs[0] and ss[1] == rs[1] and ss[4] == rs[4], (ss[0], rs[0], ss[1], rs[1], ss[4], rs[4])
    assert bits_equal(ss[3], rs[3]) == 0
    assert np.array_equal(ss[2], rs[2])
    c = center if center is not None else (rs[1] if rs[1] is not None else 0.0)
    rows = sf.grab_pulse_lens(qad, c, tol, mod, sps)
    assert np.array_equal(s_grab(ctx, qad, c, tol, mod, sps, 1, cs, ring), rows)
    q2, r2 = sf.demod_digitize(iq, noise, mod, c, tol, sps)
    q3, r3 = s_dd(ctx, iq, noise, mod, c, tol, sps, cs, ring)
    assert bits_equal(q3, q2) == 0 and np.array_equal(r3, r2)
    _, r4 = s_dd(ctx, iq, noise, mod, c, tol, sps, cs, ring, want_qad=False)
    assert np.array_equal(r4, r2)
    return rs


@pytest.mark.parametrize("tol", [0, 5, 5000])
@pytest.mark.parametrize("mod", ["FSK", "ASK"])
@pytest.mark.parametrize("cs,ring", [(TILE, 2), (3 * TILE, 3), (5 * TILE, 2)])
def test_layouts_float32(sf, ctx, cs, ring, mod, tol):
    iq = _capture(60_000 + 123, np.float32, mod)
    _check_all(sf, ctx, iq, NOISE[np.float32], mod, tol, cs, ring)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mod", ["FSK", "ASK"])
def test_dtypes(sf, ctx, dtype, mod):
    iq = _capture(3 * 7 * TILE + 1001, dtype, mod, seed=5)
    _check_all(sf, ctx, iq, NOISE[dtype], mod, 5, 7 * TILE, 3)


@pytest.mark.parametrize("n", [3, 1000, TILE, TILE + 1, 4 * TILE - 1])
def test_short_captures(sf, ctx, n):
    iq = _capture(n, np.float32, "FSK")
    _check_all(sf, ctx, iq, 0.05, "FSK", 5, 4 * TILE, 2)


@pytest.mark.parametrize("name", CAPTURES)
def test_golden(sf, ctx, name):
    g = load_golden("capture_" + name)
    mod = g["meta"]["mod"]
    if mod not in ("ASK", "FSK"):
        pytest.skip("ASK/FSK only: PSK is not streamed")
    iq = np.ascontiguousarray(g["iq"])
    sps = int(g["meta"].get("sps", 100))
    _check_all(sf, ctx, iq, float(g["noise"]), mod, 5, 3 * TILE, 3, sps=sps)


def test_no_certify_and_max_size(sf, ctx, monkeypatch):
    iq = _capture(40_000, np.float32, "FSK", seed=9)
    monkeypatch.setenv("URH_B200_CENTER_NO_CERTIFY", "1")
    rs = _check_all(sf, ctx, iq, 0.05, "FSK", 5, 3 * TILE, 2)
    assert rs[4][1] == 0
    monkeypatch.delenv("URH_B200_CENTER_NO_CERTIFY")
    _check_all(sf, ctx, iq, 0.05, "FSK", 5, 3 * TILE, 2, max_size=10_000)


def test_four_level_grab(sf, ctx):
    qad = sf.afp_demod(_capture(50_000, np.float32, "FSK", seed=2), 0.05, "FSK", 4)
    for tol in (0, 3, 3000):
        rows = sf.grab_pulse_lens(qad, 0.0, tol, "FSK", 100, bits_per_symbol=2, center_spacing=0.02)
        assert np.array_equal(s_grab(ctx, qad, 0.0, tol, "FSK", 100, 2, TILE, 3, spacing=0.02), rows)


def _budget(monkeypatch, bytes_):
    monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(int(bytes_)))


def test_shims_choose_stream(sf, monkeypatch, tmp_path):
    """through the public functions: a tiny budget streams, pinned / pageable / memory-mapped sources give the same results"""
    from urh_b200.device import PinnedArray

    iq = _capture(3 * (1 << 16) + 77, np.float32, "FSK", seed=4)
    c0, r0, q0 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100, return_qad=True)
    a0 = sf.afp_demod(iq, 0.05, "FSK", 2)
    g0 = sf.grab_pulse_lens(a0, c0, 5, "FSK", 100)
    d0 = sf.demod_digitize(iq, 0.05, "FSK", c0, 5, 100)
    pinned = PinnedArray(iq.shape, iq.dtype)
    pinned.array[:] = iq
    mm = np.memmap(tmp_path / "cap.f32", dtype=np.float32, mode="w+", shape=iq.shape)
    mm[:] = iq
    mm.flush()
    _budget(monkeypatch, 1 << 20)
    assert sf.use_stream(len(iq), iq.dtype, 5, _lib().STREAM_DEMOD_CENTER_DIGITIZE, sf.device_budget(_lib().default_context()))
    for src in (iq, pinned.array, np.memmap(tmp_path / "cap.f32", dtype=np.float32, mode="r", shape=iq.shape)):
        c1, r1, q1 = sf.demod_center_digitize(src, 0.05, "FSK", 5, 100, return_qad=True)
        assert c1 == c0 and np.array_equal(r1, r0) and bits_equal(q1, q0) == 0
        assert bits_equal(sf.afp_demod(src, 0.05, "FSK", 2), a0) == 0
        q, r = sf.demod_digitize(src, 0.05, "FSK", c0, 5, 100)
        assert bits_equal(q, d0[0]) == 0 and np.array_equal(r, d0[1])
    assert np.array_equal(sf.grab_pulse_lens(a0, c0, 5, "FSK", 100), g0)
    pinned.free()


def test_state_two_fallback(sf, ctx, monkeypatch):
    """a clean tone: detect_center's histogram has far more than 6000 bins, the device leaves the center to the host (state 2); the
    streamed step finishes it from the resident qad and the demodulator's tile table, with the same result as the resident step"""
    n = 5 * TILE + 99
    t = np.arange(n)
    x = np.exp(2j * np.pi * 0.01 * t) + 1e-5 * np.random.default_rng(1).standard_normal(n)
    iq = np.ascontiguousarray(np.stack([x.real, x.imag], axis=1).astype(np.float32))
    assert s_center(ctx, iq, 0.05, "FSK", 5, 100, TILE, 2)[0] == 2
    c0, r0, q0 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100, return_qad=True)
    _budget(monkeypatch, 1 << 20)
    c1, r1, q1 = sf.demod_center_digitize(iq, 0.05, "FSK", 5, 100, return_qad=True)
    assert c1 == c0 and np.array_equal(r1, r0) and bits_equal(q1, q0) == 0


def _stream_stats(ctx):
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_stream_stats(ctx.handle, st))
    return list(st)


def _entry_calls(ctx, iq, tol, cs, ring):
    L = _lib()
    qad = None

    def grab():
        return None, s_grab(ctx, qad, 0.0, tol, "FSK", 100, 1, cs, ring)

    def afp():
        s_afp(ctx, iq, 1000.0, "FSK", cs, ring)
        return None, None

    calls = [
        (L.STREAM_AFP_DEMOD, afp),
        (L.STREAM_DEMOD_DIGITIZE | L.STREAM_QAD_OUT, lambda: s_dd(ctx, iq, 1000.0, "FSK", 0.0, tol, 100, cs, ring)),
        (L.STREAM_DEMOD_CENTER_DIGITIZE, lambda: (None, s_center(ctx, iq, 1000.0, "FSK", tol, 100, cs, ring)[2])),
    ]
    qad = s_afp(ctx, iq, 1000.0, "FSK", cs, ring)
    calls.append((L.STREAM_GRAB_PULSE_LENS, grab))
    return calls


@pytest.mark.parametrize("tol", [0, 5])
def test_device_memory_within_footprint(sf, ctx, tol):
    """device memory in use during a streamed call (urh_mem_get_info before, the low point urh_stream_stats saw inside: after every
    chunk, after every chunk's finish and while the pulse table grows) stays within urh_stream_footprint"""
    n, cs, ring = (1 << 22) + 5, 1 << 18, 3
    iq = _capture(n, np.int16, "FSK", seed=8)
    ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 1))   # the low point is sampled only while measuring
    try:
        _footprint_calls(sf, ctx, iq, n, tol, cs, ring)
    finally:
        ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 0))


def _footprint_calls(sf, ctx, iq, n, tol, cs, ring):
    for entry, call in _entry_calls(ctx, iq, tol, cs, ring):
        ctx.sync()
        free, total = C.c_size_t(0), C.c_size_t(0)
        ctx.check(ctx.lib.urh_mem_get_info(ctx.handle, C.byref(free), C.byref(total)))
        _, rows = call()
        st = _stream_stats(ctx)
        if entry != _lib().STREAM_DEMOD_CENTER_DIGITIZE:
            assert st[1] == (n + cs - 1) // cs
        assert st[0] > 0
        used = free.value - st[0]
        assert used <= sf.stream_footprint(n, np.int16, tol, entry, cs, ring, 0 if rows is None else len(rows)), (entry, used)


@pytest.mark.parametrize("tol", [0, 5])
def test_scratch_does_not_grow_with_n(ctx, tol):
    """the digitizer's tables are sized per chunk: the most scratch-arena bytes live at once during a streamed call are the same for a
    capture 4x longer (the center entry adds only its per-tile statistics and rank prefix, < 96 B per 2048-sample tile, and one
    chunk's digitizer tables when only the longer capture has a center), also at tolerance 0, where full-length staging would need
    about 4 B/sample"""
    cs, ring = 1 << 18, 2
    peaks = {}
    for n in ((1 << 22) + 5, (1 << 24) + 5):
        iq = _capture(n, np.int16, "FSK", seed=8)
        for entry, call in _entry_calls(ctx, iq, tol, cs, ring):
            call()
            peaks.setdefault(entry, []).append(_stream_stats(ctx)[2])
    tiles = ((1 << 24) - (1 << 22)) // TILE
    for entry, (small, big) in peaks.items():
        if entry == _lib().STREAM_DEMOD_CENTER_DIGITIZE:
            # per-tile statistics and rank prefix, plus at most one chunk's digitizer tables (the digitizer is skipped when a
            # capture has no center); full-length staging would add about 4 B per added sample, 50 MB here
            assert 0 <= big - small < 96 * tiles + (2 << 20), (entry, small, big)
        else:
            assert big == small, (entry, small, big)


@pytest.mark.parametrize("name", ["fsk", "ask"])
def test_signal_and_protocol_analyzer_stream(monkeypatch, name):
    """Signal.qad and ProtocolAnalyzer.get_protocol_from_signal over a capture that does not fit the budget: demodulation and
    digitizer stream from the host, nothing of the capture stays on the device, and the messages are the resident run's"""
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.ProtocolAnalyzer import ProtocolAnalyzer
    from urh_b200.signalprocessing.Signal import Signal

    g = load_golden("capture_" + name)
    m = g["meta"]

    def run():
        s = Signal("", name)
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
    _budget(monkeypatch, 1 << 16)
    s1, pa1 = run()
    assert s1._qad_dev is None and s1.iq_array._device is None and s1.qad_device is None
    assert bits_equal(s1.qad, s0.qad) == 0
    assert pa1.plain_bits_str == pa0.plain_bits_str == m["bits"]
