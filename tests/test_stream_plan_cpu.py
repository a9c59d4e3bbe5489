"""CPU: the plan of a streamed demodulation call (the tile chunks of urh_stream_windows with URH_FILTER_TILES in the order of
urh_stream_window_schedule, urh_stream_footprint, the shims' path choice) without a device.

That no slot is rewritten before its readers is checked, for these chunks as for the windowed entries', on the host model of the
schedule in tests/test_stream_filter_plan_cpu.py."""
import ctypes as C

import numpy as np
import pytest

TILE = 2048


@pytest.fixture(scope="module")
def L():
    from urh_b200 import _lib, build

    build.build()
    return _lib


def tile_windows(L, n, cs, halo):
    lib = L.load_library()
    count = C.c_int64(0)
    args = (L.FILTER_TILES, n, n, halo, 0, cs, None, None, 0)
    assert lib.urh_stream_windows(*args, None, 0, C.byref(count)) == 0
    win = np.zeros((max(count.value, 1), 4), np.int64)
    assert lib.urh_stream_windows(*args, win.ctypes.data_as(C.c_void_p), count.value, C.byref(count)) == 0
    return win[: count.value]


def schedule(L, n, cs, ring, flags, halo):
    """ops {kind, chunk, slot, k0, k1, a, b} of the tile chunks"""
    lib = L.load_library()
    win = tile_windows(L, n, cs, halo)
    count = C.c_int64(0)
    assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), len(win), ring, flags, None, 0, C.byref(count)) == 0
    ops = np.zeros((max(count.value, 1), 7), np.int64)
    assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), len(win), ring, flags, ops.ctypes.data_as(C.c_void_p),
                                          count.value, C.byref(count)) == 0
    return ops[: count.value]


def footprint(L, n, dtype, tol, cs, ring, entry, rows=-1):
    out = C.c_int64(0)
    assert L.load_library().urh_stream_footprint(n, dtype, tol, cs, ring, entry, rows, C.byref(out)) == 0
    return out.value


@pytest.mark.parametrize("n", [1, 3, TILE - 1, TILE, TILE + 1, 5 * TILE, 7 * TILE + 3, 1_000_003])
@pytest.mark.parametrize("cs", [0, 1, TILE, 3 * TILE, 5 * TILE + 17, 1 << 18])
def test_tile_windows_cover_once_tile_aligned(L, n, cs):
    ops = schedule(L, n, cs, 2, L.STREAM_UPLOAD, 1)
    comp = ops[ops[:, 0] == 1]
    assert list(comp[:, 1]) == list(range(len(comp)))
    assert comp[0, 3] == 0 and comp[-1, 4] == n
    assert np.array_equal(comp[1:, 3], comp[:-1, 4])                     # contiguous, no overlap
    assert (comp[:, 3] % TILE == 0).all()                                  # chunks start on tile boundaries
    assert (comp[:-1, 4] - comp[:-1, 3] == comp[0, 4] - comp[0, 3]).all()  # all but the last are full
    eff = (cs if cs > 0 else 1 << 24) // TILE * TILE or TILE
    assert comp[0, 4] - comp[0, 3] == min(eff, n)
    up = ops[ops[:, 0] == 0]
    assert sorted(up[:, 1]) == list(range(len(comp)))                      # every chunk uploaded once
    assert (up[:, 3] - up[:, 5] == (up[:, 1] > 0)).all()                   # the halo (sample k0 - 1) comes with every later chunk
    assert (ops[:, 6] == ops[:, 4]).all()                                  # and nothing past the chunk's end
    no_halo = schedule(L, n, cs, 2, L.STREAM_UPLOAD, 0)
    assert (no_halo[:, 3] == no_halo[:, 5]).all()


def test_tile_schedule_rejects_bad_rings(L):
    lib = L.load_library()
    count = C.c_int64(0)
    win = tile_windows(L, 100, TILE, 1)
    for ring in (0, 1, 9):
        assert lib.urh_stream_window_schedule(win.ctypes.data_as(C.c_void_p), len(win), ring, 1, None, 0, C.byref(count)) != 0


@pytest.mark.parametrize("tol", [0, 5, 100])
@pytest.mark.parametrize("entry", [0, 1, 2, 0x12, 3])
def test_footprint_monotone(L, tol, entry):
    ns = [3, 1000, TILE, 10 * TILE + 1, 1 << 20, 1 << 24, (1 << 26) + 7, 1 << 33]
    for rows in (-1, 0):
        fp = [footprint(L, n, L.DT_F32, tol, 1 << 18, 3, entry, rows) for n in ns]
        assert all(a <= b for a, b in zip(fp, fp[1:])), fp
        res = [footprint(L, n, L.DT_F32, tol, 1 << 18, 3, entry | L.STREAM_RESIDENT, rows) for n in ns]
        assert all(a <= b for a, b in zip(res, res[1:])), res


@pytest.mark.parametrize("tol", [0, 5])
@pytest.mark.parametrize("entry", [0, 1, 2, 0x12, 1 | 0x40])
def test_footprint_flat_in_n_when_qad_not_resident(L, tol, entry):
    """apart from the pulse table (rows = 0 here) a streamed call's device memory does not grow with n, also at tolerance 0"""
    cs = 1 << 20
    fp = {footprint(L, n, L.DT_I16, tol, cs, 2, entry, 0) for n in (cs, cs + 1, 10 * cs + 3, 1 << 30, 1 << 34)}
    assert len(fp) == 1, fp
    big = footprint(L, 1 << 34, L.DT_I16, tol, cs, 2, entry, 0)
    assert big < footprint(L, 1 << 34, L.DT_I16, tol, cs, 2, entry | L.STREAM_RESIDENT, 0) / 100
    # the pulse term is all that grows: 48 bytes per budgeted row
    assert footprint(L, 1 << 30, L.DT_I16, tol, cs, 2, entry, 1000) - footprint(L, 1 << 30, L.DT_I16, tol, cs, 2, entry, 0) == \
        (0 if entry == 0 else 48 * 1000)


def test_center_footprint_grows_with_resident_qad(L):
    a = footprint(L, 1 << 28, L.DT_F32, 5, 1 << 20, 2, 3, 0)
    b = footprint(L, 1 << 29, L.DT_F32, 5, 1 << 20, 2, 3, 0)
    assert 4 * (1 << 28) <= b - a < 5 * (1 << 28)   # about 4 B/sample (qad) plus the tile tables


@pytest.mark.parametrize("entry", [0, 1, 2, 3])
def test_path_choice_at_the_budget(L, entry):
    from urh_b200.cythonext import signal_functions as sf

    for n in (5000, 1 << 22, 1 << 31):
        need = sf.stream_footprint(n, np.int8, 5, entry | L.STREAM_RESIDENT, rows=n // 64 + 1024)
        assert need == sf.stream_footprint(n, np.int8, 5, entry | L.STREAM_RESIDENT, rows=-2)
        assert sf.use_stream(n, np.int8, 5, entry, need - 1)
        assert not sf.use_stream(n, np.int8, 5, entry, need)
