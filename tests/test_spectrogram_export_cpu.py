"""CPU: the host side of the spectrogram image and FTA export against the REFERENCE's own Spectrogram class.

* The FTA record restatement (tests/fta_restatement.py) equals the file the reference's export_to_fta writes, byte for byte, with the
  reference's dB map replaced by the same seeded map (so the comparison is about the record assembly alone).
* Spectrogram.segment_bounds equals the slices the reference's create_image_segments renders, with their frame counts.
* The product raises the reference's exceptions before it opens the file or touches the device.

The reference's answers are recorded in tests/golden/ref_spectrogram_export.json (oracle/cassette.py; regenerate with
URH_RECORD_GOLDEN=1 where the reference tree exists)."""
import os

import numpy as np
import pytest

from fta_restatement import fta_bytes
from oracle.cassette import RECORD, Cassette, digest, fingerprint, same


@pytest.fixture
def cassette(request):
    c = Cassette("spectrogram_export", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ref():
    if not RECORD:
        return None
    from oracle import ref_loader
    return ref_loader.load_python_layer()


def seeded_db(frames, W, seed):
    """a fliplr'ed dB map with -inf cells (exact complex64 zeros) and a whole -inf frame"""
    rng = np.random.default_rng(seed)
    db = (rng.standard_normal((frames, W)) * 30 - 60).astype(np.float32)
    db[rng.random((frames, W)) < 0.05] = -np.inf
    if frames > 2:
        db[frames // 2] = -np.inf
    return db


def reference_fta(ref, n, W, ov, db, sample_rate, include_amplitude, path):
    """the reference's export_to_fta with its __calculate_spectrogram returning ``db``: (file bytes as uint8 or None, exception)"""
    spec = ref.Spectrogram(np.zeros(n, np.complex64), window_size=W, overlap_factor=ov)
    spec._Spectrogram__calculate_spectrogram = lambda samples: db
    if os.path.exists(path):
        os.remove(path)
    try:
        spec.export_to_fta(sample_rate, path, include_amplitude)
    except Exception as e:
        return None, (type(e).__name__, str(e), os.path.exists(path))
    with open(path, "rb") as fh:
        return np.frombuffer(fh.read(), np.uint8), None


# (n, W, overlap, sample rate): several frames, n < W (one frame), a non-integer time width, a negative sample rate
FTA_CASES = [(1000, 16, 0.5, 2e6), (5, 16, 0.5, 1e6), (777, 32, 0.3, 1.5e6), (300, 8, 0.0, 3), (1000, 16, 0.75, -2e6)]


@pytest.mark.parametrize("include_amplitude", [False, True])
@pytest.mark.parametrize("case", range(len(FTA_CASES)))
def test_fta_restatement_matches_reference_file(cassette, ref, tmp_path, case, include_amplitude):
    n, W, ov, sr = FTA_CASES[case]
    hop = W - int(ov * W)
    frames = max(1, (max(n, W) - W) // hop + 1)
    db = seeded_db(frames, W, case)
    path = str(tmp_path / "ref.fta")
    want, err = cassette.want(lambda: reference_fta(ref, n, W, ov, db, sr, include_amplitude, path))
    if err is not None:
        with pytest.raises(Exception) as e:
            fta_bytes(db, n, sr, include_amplitude)
        assert (type(e.value).__name__, str(e.value), False) == tuple(err)
        return
    mine = np.frombuffer(fta_bytes(db, n, sr, include_amplitude), np.uint8)
    assert len(mine) == W * frames * (48 if include_amplitude else 24)
    assert same(mine, want)


OVERFLOW_CASES = [(1000, 16, 0.5, 0.1), (1000, 16, 0.5, 30.0), (20, 16, 0.5, 1e-9)]   # overflow at j = 1, at a later j, n < W


@pytest.mark.parametrize("include_amplitude", [False, True])
@pytest.mark.parametrize("case", range(len(OVERFLOW_CASES)))
def test_fta_overflow_matches_reference(cassette, ref, tmp_path, case, include_amplitude):
    """a time beyond uint32: the reference raises numpy's OverflowError inside its loop and writes no file; so do the restatement
    and the product (before it opens the file or needs a device)"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n, W, ov, sr = OVERFLOW_CASES[case]
    hop = W - int(ov * W)
    frames = max(1, (max(n, W) - W) // hop + 1)
    db = seeded_db(frames, W, 7)
    path = str(tmp_path / "ref.fta")
    want, err = cassette.want(lambda: reference_fta(ref, n, W, ov, db, sr, include_amplitude, path))
    if frames == 1:   # one frame: time 0 only, never out of range
        assert err is None and same(np.frombuffer(fta_bytes(db, n, sr, include_amplitude), np.uint8), want)
        return
    assert want is None and err[0] == "OverflowError" and "out of bounds for uint32" in err[1] and err[2] is False, err
    with pytest.raises(OverflowError) as e:
        fta_bytes(db, n, sr, include_amplitude)
    assert str(e.value) == err[1]
    out = tmp_path / "product.fta"
    with pytest.raises(OverflowError) as e:
        Spectrogram(np.zeros(n, np.complex64), W, ov).export_to_fta(sr, str(out), include_amplitude)
    assert str(e.value) == err[1] and not out.exists()


def test_fta_zero_sample_rate_raises_before_any_file(cassette, ref, tmp_path):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    db = seeded_db(124, 16, 3)
    err = cassette.want(lambda: reference_fta(ref, 1000, 16, 0.5, db, 0, False, str(tmp_path / "ref.fta"))[1])
    assert err[0] == "ZeroDivisionError" and err[2] is False
    out = tmp_path / "product.fta"
    with pytest.raises(ZeroDivisionError) as e:
        Spectrogram(np.zeros(1000, np.complex64), 16, 0.5).export_to_fta(0, str(out))
    assert str(e.value) == err[1] and not out.exists()


def reference_segments(ref, n, W, ov):
    """the (start, end) pairs of the reference's create_image_segments and the frame count its stft gives each slice"""
    x = np.zeros(n, np.complex64)
    spec = ref.Spectrogram(x, window_size=W, overlap_factor=ov)
    spec.create_spectrogram_image = lambda sample_start=None, sample_end=None, **k: (sample_start, sample_end)
    out = []
    for s, e in spec.create_image_segments():
        out.append((s, min(e, n), len(spec.stft(x[s:e]))))
    return out


SEG_N = [1, 15, 16, 17, 1000, 16_000, 16_001, 24_007, 100_003, 1_048_577]


@pytest.mark.parametrize("W", [16, 64, 1000, 1024])
def test_segment_bounds_match_reference_generator(cassette, ref, W):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    for ov in (0, 0.3, 0.5, 0.75):
        for n in SEG_N:
            if W >= 1000 and n < 16:
                continue
            want = cassette.want(lambda: fingerprint(reference_segments(ref, n, W, ov)))
            mine = Spectrogram(np.zeros(n, np.complex64), W, ov).segment_bounds()
            assert fingerprint(mine) == want, (W, ov, n, mine[:4])
            assert all(0 <= s < e <= n for s, e, _ in mine)
    # the grid has captures with one and with several segments
    many = Spectrogram(np.zeros(1_048_577, np.complex64), W, 0.75).segment_bounds()
    assert len(many) > 1 or W >= 1000


def test_colormap_is_required():
    from urh_b200.signalprocessing import Spectrogram as mod

    spec = mod.Spectrogram(np.zeros(100, np.complex64), 16)
    assert mod.chosen_colormap_numpy_bgra is None
    with pytest.raises(ValueError):
        spec.create_spectrogram_image()
    with pytest.raises(ValueError):
        next(spec.create_image_segments())
    with pytest.raises(ValueError):
        spec.create_spectrogram_image(colormap=np.zeros((4, 3), np.uint8))


def test_device_samples_shape_is_checked():
    """a DeviceArray is accepted as complex64 (n,) or float32 (n, 2) only; the check needs no device memory"""
    from urh_b200.device import DeviceArray
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    fake = DeviceArray.__new__(DeviceArray)
    fake.shape, fake.dtype, fake._owns = (10, 3), np.dtype(np.float32), False
    with pytest.raises(ValueError):
        Spectrogram(fake)
    fake.shape = (10,)
    fake.dtype = np.dtype(np.complex64)
    assert Spectrogram(fake).samples is fake
