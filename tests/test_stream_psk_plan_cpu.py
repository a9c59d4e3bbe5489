"""CPU: device-memory footprints of the PSK calls (urh_stream_footprint with URH_STREAM_PSK / URH_STREAM_PSK4) and the shims' choice
between the resident and the streamed PSK path.  No device involved."""
import numpy as np
import pytest

TILE = 2048


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


def _L():
    from urh_b200 import _lib

    return _lib


ENTRIES = ("afp", "dd", "dd_qad")


def entry(kind, order):
    from urh_b200.cythonext.signal_functions import psk_entry

    L = _L()
    base = {"afp": L.STREAM_AFP_DEMOD, "dd": L.STREAM_DEMOD_DIGITIZE, "dd_qad": L.STREAM_DEMOD_DIGITIZE | L.STREAM_QAD_OUT}[kind]
    return base | psk_entry(order)


@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("kind", ENTRIES)
@pytest.mark.parametrize("dtype", (np.int8, np.int16, np.float32))
def test_monotone_in_n(sf, dtype, kind, order):
    L = _L()
    ns = [3, 8191, 8192, 100_000, 1 << 20, (1 << 20) + 1, 1 << 24, 1 << 28, 1 << 30, 1 << 33]
    for res in (0, L.STREAM_RESIDENT):
        fp = [sf.stream_footprint(n, dtype, 5, entry(kind, order) | res, 1 << 20, 2, rows=-1 if res == 0 else -2) for n in ns]
        assert all(a <= b for a, b in zip(fp, fp[1:])), (res, fp)


@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("kind", ENTRIES)
def test_streamed_flat_in_n(sf, kind, order):
    """with qad drained to the host (or digitized per chunk) the streamed footprint does not grow with n beyond the pulse table"""
    cs = 1 << 24
    fp = [sf.stream_footprint(n, np.float32, 5, entry(kind, order), cs, 2, rows=0) for n in (4 * cs, 64 * cs, 512 * cs)]
    assert fp[0] == fp[1] == fp[2], fp


@pytest.mark.parametrize("order", (2, 4, 8))
@pytest.mark.parametrize("dtype", (np.int8, np.uint16, np.float32))
def test_resident_counts_the_costas_tables(sf, dtype, order):
    """the resident PSK figure holds at least the IQ, qad and the loop's candidate samples (nbr x n float32)"""
    L = _L()
    nbr = min(order, 4)
    for n in (8192, 1_000_003, 1 << 28, 1 << 33):
        b = sf.stream_footprint(n, dtype, 0, L.STREAM_AFP_DEMOD | sf.psk_entry(order) | L.STREAM_RESIDENT, rows=-2)
        assert b >= n * 2 * np.dtype(dtype).itemsize + 4 * n + nbr * n * 4, (n, b)
        # and more than the ASK / FSK figure by at least the candidates
        plain = sf.stream_footprint(n, dtype, 0, L.STREAM_AFP_DEMOD | L.STREAM_RESIDENT, rows=-2)
        assert b - plain >= nbr * n * 4


def test_order_four_needs_more(sf):
    L = _L()
    for res in (0, L.STREAM_RESIDENT):
        for n in (1 << 20, 1 << 30):
            two = sf.stream_footprint(n, np.float32, 0, L.STREAM_AFP_DEMOD | L.STREAM_PSK | res, 1 << 24, 2, rows=-2)
            four = sf.stream_footprint(n, np.float32, 0, L.STREAM_AFP_DEMOD | L.STREAM_PSK | L.STREAM_PSK4 | res, 1 << 24, 2, rows=-2)
            assert four > two


def test_psk_flags_only_on_psk_entries(sf):
    L = _L()
    for e in (L.STREAM_GRAB_PULSE_LENS, L.STREAM_DEMOD_CENTER_DIGITIZE):
        with pytest.raises(ValueError):
            sf.stream_footprint(1 << 20, np.float32, 0, e | L.STREAM_PSK)


@pytest.mark.parametrize("order", (2, 4))
@pytest.mark.parametrize("kind", ("afp", "dd"))
def test_path_choice_flips_at_the_budget(sf, kind, order):
    """use_stream: resident exactly while the resident PSK footprint fits the budget"""
    L = _L()
    n = 3 * (1 << 20) + 5
    e = entry(kind, order)
    need = sf.stream_footprint(n, np.int16, 5, e | L.STREAM_RESIDENT, rows=-2)
    assert not sf.use_stream(n, np.int16, 5, e, need)
    assert sf.use_stream(n, np.int16, 5, e, need - 1)
    # the PSK figure is larger than the ASK / FSK one: a budget between the two streams PSK only
    plain = sf.stream_footprint(n, np.int16, 5, e & ~(L.STREAM_PSK | L.STREAM_PSK4) | L.STREAM_RESIDENT, rows=-2)
    assert plain < need
    assert sf.use_stream(n, np.int16, 5, e, plain) and not sf.use_stream(n, np.int16, 5, e & 0xF, plain)


def test_shim_entries_follow_the_order(sf):
    """psk_entry maps a loop order to the footprint flags: order 2 (and the serial orders 1 and 3) -> PSK, 4 and above -> PSK4"""
    L = _L()
    assert sf.psk_entry(2) == L.STREAM_PSK
    assert sf.psk_entry(3) == L.STREAM_PSK
    assert sf.psk_entry(4) == sf.psk_entry(8) == L.STREAM_PSK | L.STREAM_PSK4
