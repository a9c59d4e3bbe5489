"""CPU suite for the signal view: the numpy restatement of path_creator.create_path (tests/path_restatement.py) is pinned byte for
byte to the reference's compiled path_creator.pyx.  The reference's answers (sha256 of the exact stream bytes) are recorded in
tests/golden/ref_path_creator.json and replayed; where oracle/build_ref_path_creator.py has built the reference, the comparison
also runs live."""
import numpy as np
import pytest

from oracle.cassette import Cassette
import path_restatement as R
import qt_fake


def _reference():
    try:
        from oracle import build_ref_path_creator

        return build_ref_path_creator.load()
    except Exception:
        return None


def _reference_streams(ref, samples, start, end, ranges, ppp):
    import urh.settings

    old = urh.settings.PIXELS_PER_PATH
    urh.settings.PIXELS_PER_PATH = ppp
    try:
        with qt_fake.installed(ref):
            paths = ref.create_path(samples, start, end, ranges)
    finally:
        urh.settings.PIXELS_PER_PATH = old
    return [p.stream or b"" for p in paths]


def test_restatement_pinned_to_recorded_reference():
    cas = Cassette("path_creator", "test_restatement_pinned_to_recorded_reference")
    ref = cas.make(_reference) if cas.recording else None
    bad = []
    for cid, x, start, end, ranges, ppp in R.all_cases():
        mine = R.digest(R.create_path_streams(x, start, end, ranges, ppp)[0])
        want = cas.want(lambda: [cid, R.digest(_reference_streams(ref, x, start, end, ranges, ppp))])
        if want != [cid, mine]:
            bad.append(cid)
    cas.close()
    assert not bad, bad


def test_float64_raises_type_error_as_recorded():
    cas = Cassette("path_creator", "test_float64_raises_type_error_as_recorded")
    ref = cas.make(_reference) if cas.recording else None

    def ref_error():
        try:
            _reference_streams(ref, np.zeros(100), 0, 100, None, 5000)
        except Exception as e:
            return type(e).__name__
        return None

    assert cas.want(ref_error) == "TypeError"
    cas.close()
    with pytest.raises(TypeError):
        R.create_path_streams(np.zeros(100), 0, 100)
    from urh_b200.cythonext import path_creator as pc

    with pytest.raises(TypeError):   # rejected before any device work
        pc.create_path_streams(np.zeros(100), 0, 100)


@pytest.mark.skipif(_reference() is None, reason="reference path_creator not built here")
def test_restatement_equals_live_reference():
    ref = _reference()
    for cid, x, start, end, ranges, ppp in R.all_cases():
        assert R.create_path_streams(x, start, end, ranges, ppp)[0] == _reference_streams(ref, x, start, end, ranges, ppp), cid


def test_host_array_to_qpath_matches_restatement():
    from urh_b200.cythonext import path_creator as pc

    y = np.array([0.0, -0.0, np.inf, -np.inf, 1.5], dtype=np.float32)
    y = np.concatenate([y, np.array([0x7fc12345, 0xff800001, 1], dtype=np.uint32).view(np.float32)])
    x = np.arange(10, 10 + len(y), dtype=np.int64)
    for d in R.DTYPES:
        yy = y if d is np.float32 else np.array([0, 1, -1, 127, 255, -128, 3, 9], dtype=np.int64).astype(d)
        assert pc.qpath_stream(x, yy) == R.stream(x, yy)
    assert pc.qpath_stream(x[:0], y[:0]) == b""
    with qt_fake.installed():
        path = pc.array_to_QPath(x, y)
        empty = pc.array_to_QPath(x[:0], y[:0])
    assert path.stream == R.stream(x, y) and empty.stream is None


@pytest.mark.skipif(_reference() is None, reason="reference path_creator not built here")
def test_host_array_to_qpath_equals_live_reference():
    from urh_b200.cythonext import path_creator as pc

    ref = _reference()
    for d in R.DTYPES:
        y = R.random_samples(d, 257, 5)
        x = np.arange(3, 260, dtype=np.int64)
        with qt_fake.installed(ref):
            assert ref.array_to_QPath(x, y).stream == pc.qpath_stream(x, y)


def test_create_path_without_qt_raises_import_error(monkeypatch):
    import sys

    from urh_b200.cythonext import path_creator as pc

    for name in ("PyQt6", "PyQt6.QtCore", "PyQt6.QtGui"):
        monkeypatch.setitem(sys.modules, name, None)   # as if Qt were not installed
    with pytest.raises(ImportError):
        pc.create_path(np.zeros(10, np.float32), 0, 10)
