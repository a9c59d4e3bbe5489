"""GPU: the auto-interpretation steps from a host capture streamed through the device (urh_noise_chunk_stats_iq_stream,
urh_segment_messages_iq_stream, urh_convert_iq_stream; DESIGN.md §4.11) give the resident calls' results word for word, and
Signal(path) -> auto_detect() -> get_protocol_from_signal() under a device budget below every resident footprint gives what the
unconstrained run gives."""
import ctypes as C

import numpy as np
import pytest

from autointerp_cases import IQ_DTYPES, noise_iq_cases

pytestmark = pytest.mark.gpu

TILE = 2048
GOLDEN = ["capture_FSK10", "capture_ask", "capture_ask_short", "capture_enocean", "capture_esaver", "capture_fsk", "capture_homematic",
          "capture_psk_gen_noisy", "capture_two_participants"]


def _lib():
    from urh_b200 import _lib as L

    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def golden(name):
    import os

    return np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))["iq"]


def chunking(n):
    chunksize = max(1, int(n * 1 / 100))
    return chunksize, n // chunksize


def to_dtype(x, dt):
    """complex samples of magnitude <= 1 as an (n, 2) capture of dtype dt"""
    iq = np.stack([x.real, x.imag], 1)
    if dt == np.float32:
        return np.ascontiguousarray(iq.astype(np.float32))
    info = np.iinfo(dt)
    mid = (int(info.max) + int(info.min) + 1) // 2
    return np.ascontiguousarray(np.clip(np.rint(iq * (int(info.max) - mid) * 0.99) + mid, info.min, info.max).astype(dt))


# ---- noise-chunk statistics --------------------------------------------------------------------------------------------------------
def noise_resident(ctx, iq):
    from urh_b200.device import to_device

    n = len(iq)
    cs, nch = chunking(n)
    d = to_device(iq, ctx)
    s, m = np.empty(nch), np.empty(nch)
    ctx.check(ctx.lib.urh_noise_chunk_stats_iq(ctx.handle, C.c_void_p(d.ptr), _lib().dtype_code(iq.dtype), n, cs, nch, _ptr(s), _ptr(m)))
    return s, m


def noise_streamed(ctx, iq, chunk, ring):
    n = len(iq)
    cs, nch = chunking(n)
    s, m = np.full(nch, np.nan), np.full(nch, np.nan)
    ctx.check(ctx.lib.urh_noise_chunk_stats_iq_stream(ctx.handle, _ptr(iq), _lib().dtype_code(iq.dtype), n, cs, nch, chunk, ring,
                                                      _ptr(s), _ptr(m)))
    return s, m


def same_words(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def noise_chunks_for(n):
    per = -(-chunking(n)[0] // 64)
    return sorted({per, 3 * per + 1, max(1, per // 2), 1 << 14})


@pytest.mark.parametrize("dtype", IQ_DTYPES)
@pytest.mark.parametrize("ring", [2, 3])
def test_noise_stream_every_dtype(ctx, dtype, ring):
    rng = np.random.default_rng(11)
    for n in (4, 5, 99, 101, 6401, 123_457):
        x = np.exp(2j * np.pi * rng.random(n)) * np.where(np.arange(n) < n // 2, 0.9, 0.05)
        iq = to_dtype(x, dtype)
        ref = noise_resident(ctx, iq)
        for chunk in noise_chunks_for(n):
            got = noise_streamed(ctx, iq, chunk, ring)
            assert same_words(got[0], ref[0]) and same_words(got[1], ref[1]), (n, chunk)


def test_noise_stream_case_matrix_and_golden(ctx):
    cases = list(noise_iq_cases()) + [(name, golden(name)) for name in GOLDEN]
    for name, iq in cases:
        iq = np.ascontiguousarray(iq)
        if len(iq) <= 3:
            continue
        ref = noise_resident(ctx, iq)
        for chunk in noise_chunks_for(len(iq)):
            got = noise_streamed(ctx, iq, chunk, 2)
            assert same_words(got[0], ref[0]) and same_words(got[1], ref[1]), (name, chunk)


# ---- segmentation ------------------------------------------------------------------------------------------------------------------------
def seg_resident(ctx, iq, thr):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.cythonext import util
    from urh_b200.device import to_device

    return AI.segment_messages_from_magnitudes(util.get_magnitudes(to_device(iq, ctx)), thr)


def seg_streamed(ctx, iq, thr, chunk, ring=2):
    k = C.c_int64(-1)
    ctx.check(ctx.lib.urh_segment_messages_iq_stream(ctx.handle, _ptr(iq), _lib().dtype_code(iq.dtype), len(iq), float(thr), chunk, ring,
                                                     C.byref(k)))
    seg = np.empty((k.value, 2), np.int64)
    ctx.check(ctx.lib.urh_fetch_segments(ctx.handle, _ptr(seg), k.value))
    return [(int(a), int(b)) for a, b in seg]


def from_levels(levels, dtype, rng):
    """a capture whose magnitude is `levels` (0.9 above, 0.05 below a threshold of 0.5), random phase"""
    return to_dtype(levels * np.exp(2j * np.pi * rng.random(len(levels))), dtype)


def runs(*pairs):
    """levels from (length, above) runs"""
    return np.concatenate([np.full(length, 0.9 if above else 0.05) for length, above in pairs])


def seg_cases():
    yield "silence and message longer than several chunks", runs((5 * TILE + 17, 0), (7 * TILE + 3, 1), (4 * TILE, 0), (9, 1), (3 * TILE + 1, 0))
    # the 10th consecutive sample of a run falls on a chunk edge (tiles of one chunk: chunk edges at every multiple of 2048)
    yield "10th above sample on the edge", runs((TILE - 9, 0), (300, 1), (TILE, 0))
    yield "10th below sample on the edge", runs((100, 0), (2 * TILE - 109, 1), (500, 0), (TILE, 1))
    yield "9 and 10 across the edge", runs((TILE - 5, 0), (9, 1), (10, 0), (TILE - 14, 1), (TILE + 3, 0))
    yield "starts above, ends inside a message", runs((3 * TILE + 5, 1), (700, 0), (2 * TILE + 11, 1))
    yield "starts above, ends in a short silence", runs((TILE + 1, 1), (9, 0))
    yield "shorter than a chunk", runs((100, 0), (400, 1), (333, 0))
    rng = np.random.default_rng(5)
    lv = np.repeat(rng.random(4000) < 0.5, rng.integers(1, 40, 4000))
    yield "random runs", np.where(lv, 0.9, 0.05)


@pytest.mark.parametrize("dtype", IQ_DTYPES)
def test_segment_stream_matches_resident(ctx, dtype):
    rng = np.random.default_rng(7)
    for name, levels in seg_cases():
        iq = from_levels(levels, dtype, rng)
        thr = 0.5 * (float(np.iinfo(dtype).max) if dtype != np.float32 else 1.0)
        ref = seg_resident(ctx, iq, thr)
        assert ref or dtype in (np.uint8, np.uint16), name   # unsigned samples are not centred: every magnitude is large
        for chunk in (TILE, 3 * TILE, 1 << 20):
            for ring in (2, 3):
                assert seg_streamed(ctx, iq, thr, chunk, ring) == ref, (name, chunk, ring)


def test_segment_stream_golden(ctx):
    from urh_b200.ainterpretation import AutoInterpretation as AI

    for name in GOLDEN:
        iq = np.ascontiguousarray(golden(name))
        thr = AI.detect_noise_level_iq(iq)
        assert seg_streamed(ctx, iq, thr, TILE) == seg_resident(ctx, iq, thr), name


def test_segment_shim_streams_once_past_the_first_buffer(ctx, monkeypatch):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.cythonext import signal_functions as sf

    nmsg = (1 << 16) + 5   # more messages than a 2^16-pair buffer holds
    levels = np.tile(runs((10, 1), (10, 0)), nmsg)
    iq = from_levels(levels, np.float32, np.random.default_rng(3))
    ref = seg_resident(ctx, iq, 0.5)
    assert len(ref) == nmsg
    calls = []
    fn = ctx.lib.urh_segment_messages_iq_stream
    monkeypatch.setattr(ctx.lib, "urh_segment_messages_iq_stream", lambda *a: calls.append(1) or fn(*a))
    monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(1 << 20))
    monkeypatch.setattr(sf, "STREAM_CHUNK", 1 << 16)
    assert AI.segment_messages_iq(iq, 0.5) == ref
    assert len(calls) == 1


# ---- conversion ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("src, dst", [(np.uint8, np.int8), (np.uint16, np.int16), (np.int8, np.float32), (np.float32, np.int16),
                                      (np.int16, np.uint8)])
def test_convert_stream_matches_resident(ctx, src, dst):
    from urh_b200.signalprocessing.IQArray import IQArray

    rng = np.random.default_rng(1)
    for n in (1, 1000, 100_003):
        if src == np.float32:
            x = np.ascontiguousarray((rng.random((n, 2)) * 2.2 - 1.1).astype(np.float32))
        else:
            info = np.iinfo(src)
            x = rng.integers(info.min, int(info.max) + 1, (n, 2)).astype(src)
        ref = IQArray(x.copy()).convert_to_device(dst).get()
        for chunk in (1, 777, 1 << 14):
            out = np.empty((n, 2), dst)
            ctx.check(ctx.lib.urh_convert_iq_stream(ctx.handle, _ptr(x), _lib().dtype_code(src), _ptr(out), _lib().dtype_code(dst), n,
                                                    chunk, 2))
            assert np.array_equal(out.view(np.uint8), ref.view(np.uint8)), (n, chunk)


# ---- the shims under a low device budget -----------------------------------------------------------------------------------------------
STREAMED = ("urh_noise_chunk_stats_iq_stream", "urh_segment_messages_iq_stream", "urh_convert_iq_stream", "urh_afp_demod_stream",
            "urh_afp_demod_psk_stream")


@pytest.fixture
def low_budget(monkeypatch, ctx):
    """set_low(): a device budget below every resident call's footprint, and small chunks so that every streamed call has several.
    streamed: how often each streamed entry was called (the library's functions wrapped for the test)."""
    from urh_b200.cythonext import signal_functions as sf

    streamed = {}
    for name in STREAMED:
        fn = getattr(ctx.lib, name)

        def wrapped(*args, _fn=fn, _name=name):
            streamed[_name] = streamed.get(_name, 0) + 1
            return _fn(*args)
        monkeypatch.setattr(ctx.lib, name, wrapped)

    def set_low():
        monkeypatch.setenv("URH_B200_DEVICE_BUDGET", str(1 << 20))
        monkeypatch.setattr(sf, "STREAM_CHUNK", 1 << 14)
        monkeypatch.setattr(sf, "FILTER_STREAM_CHUNK", 1 << 14)
        monkeypatch.setattr(sf, "PSK_STREAM_CHUNK", 1 << 15)
    set_low.streamed = streamed
    return set_low


def test_from_file_cu8_streams(ctx, low_budget, tmp_path):
    from urh_b200.signalprocessing.IQArray import IQArray

    raw = np.random.default_rng(4).integers(0, 256, (100_001, 2)).astype(np.uint8)
    path = tmp_path / "x.cu8"
    raw.tofile(path)
    ref = IQArray.from_file(str(path))
    assert not low_budget.streamed
    low_budget()
    got = IQArray.from_file(str(path))
    assert low_budget.streamed.get("urh_convert_iq_stream") == 1
    assert got.dtype == np.int8 and np.array_equal(got._peek(), ref._peek())


def synthetic_capture():
    """several chunks of FSK, OOK and PSK bursts separated by noise"""
    rng = np.random.default_rng(21)
    sps, parts = 50, []
    for mod in ("FSK", "OOK", "PSK"):
        for _ in range(3):
            bits = np.repeat(rng.integers(0, 2, 120), sps)
            t = np.arange(len(bits))
            if mod == "FSK":
                x = np.exp(1j * np.cumsum(np.where(bits > 0, 0.3, -0.3)))
            elif mod == "OOK":
                x = np.where(bits > 0, 0.9, 0.0) * np.exp(0.2j * t)
            else:
                x = np.exp(1j * (0.1 * t + np.pi * bits))
            parts.append(0.8 * x)
            parts.append(np.zeros(3000))
    x = np.concatenate(parts)
    x = x + 0.01 * (rng.standard_normal(len(x)) + 1j * rng.standard_normal(len(x)))
    return to_dtype(x, np.float32)


def chain(path):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.signalprocessing.ProtocolAnalyzer import ProtocolAnalyzer
    from urh_b200.signalprocessing.Signal import Signal

    s = Signal(str(path), "t")
    host = s.iq_array._peek()
    out = {"noise": s.noise_threshold,
           "estimate_given": AI.estimate(host.copy(), noise=s.noise_threshold, modulation="FSK"),
           "estimate_none": AI.estimate(host.copy())}
    out["detected"] = s.auto_detect(detect_modulation=True, detect_noise=False)
    out["params"] = (s.modulation_type, s.center, s.tolerance, s.samples_per_symbol)
    pa = ProtocolAnalyzer(s)
    pa.get_protocol_from_signal()
    out["messages"] = [(m.plain_bits_str, m.pause, list(np.asarray(m.bit_sample_pos))) for m in pa.messages]
    return out


def test_chain_under_low_budget(ctx, low_budget, tmp_path):
    ext = {np.dtype(np.float32): ".complex", np.dtype(np.int8): ".complex16s", np.dtype(np.int16): ".complex32s"}
    captures = {name: golden(name) for name in GOLDEN}
    captures["synthetic"] = synthetic_capture()
    paths = {}
    for name, iq in captures.items():
        paths[name] = tmp_path / (name + ext[iq.dtype])
        np.ascontiguousarray(iq).tofile(paths[name])
    ref = {name: chain(p) for name, p in paths.items()}
    assert not low_budget.streamed, low_budget.streamed   # captures that fit keep the resident path
    low_budget()
    for name, p in paths.items():
        assert chain(p) == ref[name], name
    for entry in ("urh_noise_chunk_stats_iq_stream", "urh_segment_messages_iq_stream", "urh_afp_demod_stream"):
        assert low_budget.streamed.get(entry, 0) > 0, (entry, low_budget.streamed)


# ---- device memory -------------------------------------------------------------------------------------------------------------------
def _stream_stats(ctx):
    st = (C.c_int64 * 3)()
    ctx.check(ctx.lib.urh_stream_stats(ctx.handle, st))
    return list(st)


def _runs(ctx, n, chunk):
    rng = np.random.default_rng(9)
    x = np.exp(2j * np.pi * rng.random(n)) * np.where((np.arange(n) // 5000) % 3 == 0, 0.9, 0.05)
    iq = to_dtype(x, np.int16)
    cs, nch = chunking(n)
    from urh_b200.cythonext import signal_functions as sf

    L = _lib()
    return [
        (sf.filter_footprint(L.FILTER_NOISE, n, 0, iq.dtype, cs, nch, chunk, 3), lambda: noise_streamed(ctx, iq, chunk, 3)),
        (sf.filter_footprint(L.FILTER_CONVERT, n, n, iq.dtype, L.DT_F32, 0, chunk, 3),
         lambda: ctx.check(ctx.lib.urh_convert_iq_stream(ctx.handle, _ptr(iq), L.DT_I16, _ptr(np.empty((n, 2), np.float32)), L.DT_F32, n,
                                                         chunk, 3))),
        (sf.stream_footprint(n, iq.dtype, 0, L.STREAM_SEGMENT_MESSAGES, chunk, 3), lambda: seg_streamed(ctx, iq, 16000.0, chunk, 3)),
    ]


def test_device_memory_within_footprint(ctx):
    n, chunk = (1 << 22) + 5, 1 << 18
    ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 1))   # the low point is sampled only while measuring
    try:
        for footprint, call in _runs(ctx, n, chunk):
            ctx.sync()
            free, total = C.c_size_t(0), C.c_size_t(0)
            ctx.check(ctx.lib.urh_mem_get_info(ctx.handle, C.byref(free), C.byref(total)))
            call()
            st = _stream_stats(ctx)
            assert st[0] > 0 and st[1] > 1, st
            assert free.value - st[0] <= footprint, (footprint, free.value - st[0])
    finally:
        ctx.check(ctx.lib.urh_set_profiling(ctx.handle, 0))


def test_arena_peak_independent_of_n(ctx):
    chunk = 1 << 18
    peaks = []
    for n in (1 << 22, 1 << 24):   # the segmentation's peak is its largest chunk's: one full chunk's segmenter pass in both
        peaks.append([(call(), _stream_stats(ctx)[2])[1] for _, call in _runs(ctx, n, chunk)])
    assert peaks[0] == peaks[1], peaks
