"""GPU: IQArray.export_to_sub (urh_sub_export, subexport.cu) writes the restatement's file (tests/sub_restatement.py) byte for byte:
on the CPU suite's whole matrix (pinned there to the reference's own files), and on captures of 2^20 .. 2^26 samples built to stress
the tiled chain: OOK-like long runs, uniform noise over all 256 values, an armed value that never recurs, dense length-1 / length-2
runs, and runs of every length around the tile size at every offset.  A host capture and a capture already cached on the device give
the same file.  A host capture over the device budget streams through the ring (rings of 2 and 8 slots, chunk edges inside runs and
inside skips, the body written piece by piece) and gives the same file, with its arena peak under urh_sub_export_footprint.  A .sub
file loaded with Signal exports to the reference's own file, and the error cases raise the reference's exact exceptions."""
import numpy as np
import pytest

from sub_restatement import sub_file, u8_column
from test_sub_export_cpu import CASES, ERROR_CASES

pytestmark = pytest.mark.gpu

TILE = 2048


def export_bytes(iq, tmp_path, **kw):
    path = tmp_path / "out.sub"
    iq.export_to_sub(str(path), **kw)
    return path.read_bytes()


def capture(col, dtype, seed=0):
    """an (n, 2) capture whose convert_to(uint8)[:, 0] is col"""
    rng = np.random.default_rng(seed)
    col = np.asarray(col, np.uint8)
    if dtype == np.uint8:
        i = col
    elif dtype == np.int8:
        i = (col.astype(np.int16) - 128).astype(np.int8)
    else:
        i = ((col.astype(np.float32) + 0.5) / 127 - 1).astype(np.float32)
    q = np.zeros(len(col), dtype)
    data = np.stack([i, q], axis=1)
    assert np.array_equal(u8_column(data), col)
    return data


def ook(n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 6000, n // 1000 + 2)
    lengths[rng.random(len(lengths)) < 0.01] = 1
    vals = np.where(np.arange(len(lengths)) % 2 == 0, 0, 255).astype(np.uint8)
    other = rng.random(len(lengths)) < 0.01
    vals[other] = rng.integers(0, 256, int(other.sum()))
    return np.repeat(vals, lengths)[:n]


def noise(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n).astype(np.uint8)


def never_recurs(n, seed):
    rng = np.random.default_rng(seed)
    col = np.repeat(rng.integers(0, 2, n // 3 + 1).astype(np.uint8) + 10, 3)[:n]
    col[0] = 99
    return col


def dense(n, seed):
    rng = np.random.default_rng(seed)
    return np.repeat(rng.integers(20, 23, n).astype(np.uint8), rng.integers(1, 3, n))[:n]


def tile_edges(n, seed):
    """runs of TILE - 1, TILE, TILE + 1 and short runs, so that run starts fall at every offset of a tile"""
    rng = np.random.default_rng(seed)
    pattern = np.array([TILE - 1, TILE, TILE + 1, 1, 2, 3, 2 * TILE + 1, 1, 5, TILE - 2, 7, 1])
    lengths = np.resize(pattern, n // 1000 + 16)
    vals = rng.integers(0, 4, len(lengths)).astype(np.uint8) * 60
    return np.repeat(vals, lengths)[:n]


@pytest.mark.parametrize("name", sorted(CASES))
def test_matrix_matches_restatement(tmp_path, name):
    from urh_b200.signalprocessing.IQArray import IQArray

    data, kw = CASES[name]
    assert export_bytes(IQArray(data.copy()), tmp_path, **kw) == sub_file(u8_column(data), **kw)


def recorded(test):
    """the reference's answers recorded by tests/test_sub_export_cpu.py::<test>"""
    from oracle.cassette import Cassette

    return Cassette("sub_export", test).values


@pytest.mark.parametrize("name", sorted(ERROR_CASES))
def test_errors_leave_no_file(tmp_path, name):
    from urh_b200.signalprocessing.IQArray import IQArray

    data, skip = ERROR_CASES[name]
    want, err = recorded("test_errors_match_reference_without_file[%s]" % name)[0]
    path = tmp_path / "x.sub"
    with pytest.raises(Exception) as e:
        IQArray(data, skip_conversion=skip).export_to_sub(str(path))
    assert (type(e.value).__name__, str(e.value), path.exists()) == tuple(err)


def test_one_column_capture(tmp_path):
    """an (n, 1) capture wrapped with skip_conversion: the reference reads its column 0"""
    from urh_b200.signalprocessing.IQArray import IQArray

    col = dense(5000, 3)
    data = capture(col, np.int8)[:, :1].copy()
    assert export_bytes(IQArray(data, skip_conversion=True), tmp_path) == sub_file(col)


def test_sub_fixture_round_trip_on_device(tmp_path):
    """a .sub file loaded with Signal and exported on the device: the reference's own file (recorded on the CPU)"""
    from urh_b200 import settings
    from urh_b200.signalprocessing.Signal import Signal

    path = tmp_path / "remote.sub"
    path.write_text("Filetype: Flipper SubGhz RAW File\nVersion: 1\nFrequency: 433920000\nPreset: FuriHalSubGhzPresetOok650Async\n"
                    "Protocol: RAW\nRAW_Data: 300 -900 300 -300 900 -9000 1 -1 2 -2\nRAW_Data: 450 -450 1350 -100\n")
    settings.write("default_noise_threshold", "3")
    try:
        sig = Signal(str(path), "t")
    finally:
        settings.write("default_noise_threshold", "automatic")
    from oracle.cassette import same

    want = recorded("test_sub_fixture_round_trip")[0]
    assert same(np.frombuffer(export_bytes(sig.iq_array, tmp_path), np.uint8), want)


LARGE = [("ook", ook, 1 << 20, np.float32), ("ook", ook, 1 << 26, np.int8), ("noise", noise, 1 << 20, np.uint8),
         ("noise", noise, 1 << 24, np.float32), ("never_recurs", never_recurs, 1 << 22, np.int8), ("dense", dense, 1 << 20, np.uint8),
         ("tile_edges", tile_edges, 1 << 22, np.float32), ("tile_edges", tile_edges, (1 << 22) + 777, np.uint8)]


@pytest.mark.parametrize("case", range(len(LARGE)), ids=["%s_%d_%s" % (c[0], c[2], np.dtype(c[3]).name) for c in LARGE])
def test_large_matches_restatement(tmp_path, case):
    from urh_b200.signalprocessing.IQArray import IQArray

    _, make, n, dtype = LARGE[case]
    col = make(n, case)
    data = capture(col, dtype, case)
    assert export_bytes(IQArray(data), tmp_path) == sub_file(col)


def test_tile_edge_offsets(tmp_path):
    """one long run ending at every offset around a tile edge, with the armed value skipping across it"""
    from urh_b200.signalprocessing.IQArray import IQArray

    for end in list(range(TILE - 3, TILE + 4)) + [3 * TILE - 1, 3 * TILE, 3 * TILE + 1]:
        for head in ([], [5], [5, 6], [5, 5]):
            col = np.r_[head, np.full(end - len(head), 200), [5, 7, 7, 5, 5], np.full(TILE + 1, 9), [5]].astype(np.uint8)
            assert export_bytes(IQArray(capture(col, np.uint8)), tmp_path) == sub_file(col), (end, head)


def test_cached_device_capture_gives_same_file(tmp_path):
    from urh_b200.signalprocessing.IQArray import IQArray

    col = noise(1 << 20, 7)
    col[: 1 << 19] = ook(1 << 19, 8)
    data = capture(col, np.float32)
    iq = IQArray(data.copy(), _owned=True)
    dev = iq.device()
    assert iq.device() is dev   # cached: the export reads it without another upload
    a = export_bytes(iq, tmp_path)
    assert iq.device() is dev
    b = export_bytes(IQArray(data), tmp_path)
    assert a == b == sub_file(col)


def stream_stats():
    import ctypes

    from urh_b200 import _lib

    ctx = _lib.default_context()
    out = (ctypes.c_int64 * 3)()
    ctx.check(ctx.lib.urh_stream_stats(ctx.handle, out))
    return list(out)


def streamed_footprint(n, dtype, chunk, ring):
    import ctypes

    from urh_b200 import _lib

    fp = ctypes.c_int64(0)
    assert _lib.load_library().urh_sub_export_footprint(n, _lib.dtype_code(dtype), 1, chunk, ring, ctypes.byref(fp)) == 0
    return fp.value


def skips_across_chunks(n, chunk):
    """long runs ending 1 before, at and 1 after every chunk edge, one-sample runs whose value recurs only a chunk later"""
    parts = []
    k = 0
    while sum(map(len, parts)) < n:
        parts.append(np.full(chunk - 1 + (k % 3), 40 + k % 2, np.uint8))
        parts.append(np.array([200 + k % 5, 7, 7], np.uint8))
        k += 1
    return np.concatenate(parts)[:n]


STREAM_CASES = [(2, 3 * TILE, np.float32, "tile_edges"), (8, 3 * TILE, np.int16, "skips"), (2, 5 * TILE, np.uint8, "noise"),
                (8, 7 * TILE, np.int8, "ook"), (2, 1 << 18, np.float32, "skips")]


@pytest.mark.parametrize("case", range(len(STREAM_CASES)),
                         ids=["ring%d_chunk%d_%s_%s" % (c[0], c[1], np.dtype(c[2]).name, c[3]) for c in STREAM_CASES])
def test_streamed_matches_resident(tmp_path, monkeypatch, case):
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.IQArray import IQArray

    ring, chunk, dtype, kind = STREAM_CASES[case]
    n = 40 * chunk + 777
    col = {"tile_edges": lambda: tile_edges(n, case), "skips": lambda: skips_across_chunks(n, chunk),
           "noise": lambda: noise(n, case), "ook": lambda: ook(n, case)}[kind]()
    if dtype == np.int16:
        data = np.stack([((col.astype(np.int32) << 8) - 32768).astype(np.int16), np.zeros(n, np.int16)], axis=1)
    else:
        data = capture(col, dtype, case)
    assert np.array_equal(u8_column(data), col)
    want = sub_file(col)
    resident = export_bytes(IQArray(data), tmp_path)
    monkeypatch.setattr(sf, "FILTER_STREAM_CHUNK", chunk)
    monkeypatch.setattr(sf, "STREAM_RING", ring)
    monkeypatch.setenv("URH_B200_DEVICE_BUDGET", "1")
    streamed = export_bytes(IQArray(data), tmp_path)
    stats = stream_stats()
    assert stats[1] == -(-n // chunk)   # it streamed: one ring computation per chunk
    assert 0 < stats[2] <= streamed_footprint(n, dtype, chunk, ring)
    assert streamed == resident == want


def test_streamed_footprint_below_resident():
    import ctypes

    from urh_b200 import _lib

    lib = _lib.load_library()
    for n in (1, 2048, 1 << 20, 1 << 30, 1 << 34):
        for dt in (_lib.DT_U8, _lib.DT_F32):
            fp = [ctypes.c_int64(0), ctypes.c_int64(0)]
            for streamed in (0, 1):
                assert lib.urh_sub_export_footprint(n, dt, streamed, 1 << 24, 2, ctypes.byref(fp[streamed])) == 0
            if n >= 1 << 30:
                assert fp[1].value < fp[0].value
