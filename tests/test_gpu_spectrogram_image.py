"""GPU: spectrogram images (urh_spectrogram_bgra: STFT -> dB -> colormap in one launch for every segment) and the streamed FTA
export (urh_fta_records), against the two device stages they fuse, the reference's own Spectrogram class and the FTA restatement.

Paths (DESIGN 4.6): powers of two 128 .. 4096: k_stft_r16 mode 2;  everything else: urh_spectrogram_db's kernels + k_bgra_place
(composed)."""
import ctypes as C
import os

import numpy as np
import pytest

from fta_restatement import fta_bytes

pytestmark = pytest.mark.gpu

OVERLAPS = [0, 0.3, 0.5, 0.75]
RANGES = [(-140, 10), (-80, 10), (-60, -60)]
WINDOW_SIZES = [128, 256, 512, 1024, 2048, 4096, 1000, 1001]


def colormap(entries, seed=0):
    """distinct BGRA entries (so that a pixel names its index)"""
    rng = np.random.default_rng(seed)
    idx = np.arange(entries, dtype=np.uint32) * 2654435761 % (1 << 24)
    cmap = np.empty((entries, 4), np.uint8)
    cmap[:, 0], cmap[:, 1], cmap[:, 2] = idx & 255, (idx >> 8) & 255, idx >> 16
    cmap[:, 3] = rng.integers(0, 256, entries)
    return cmap


CMAPS = {L: colormap(L, L) for L in (256, 1024, 1025)}


def capture(n, W, seed=1):
    """a tone + DC, noise in the second half, and 2 W exact zeros (frames of zeros: -inf)"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = (0.25 - 0.5j) + 2.0 * np.exp(2j * np.pi * 0.1937 * t)
    x[n // 2:] += 1e-3 * (rng.standard_normal(n - n // 2) + 1j * rng.standard_normal(n - n // 2))
    x[n // 2 + W // 2: n // 2 + W // 2 + 2 * W] = 0
    return x.astype(np.complex64)


def lengths(W, hop):
    return sorted({1, W - 1, W, W + 1, W + hop, W + 7 * hop + 3, W + 20 * hop + hop // 2})


def composed(spec, x, transpose, cmap):
    """the reference's composition with this library's two device stages: apply_bgra_lookup(dB map) (transpose: of flipud(dB.T))"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    db = spec.calculate_spectrogram(x)
    data = np.flipud(db.T) if transpose else db
    return Spectrogram.apply_bgra_lookup(data, cmap, spec.data_min, spec.data_max)


@pytest.mark.parametrize("W", WINDOW_SIZES)
def test_fused_image_equals_db_map_then_lookup(W):
    """create_spectrogram_image == urh_bgra_lookup(urh_spectrogram_db(...)) bit for bit on the kernel that serves W, every overlap,
    1 .. ~20 frames (n < W included), both layouts, three (min, max) ranges (one with min = max) and colormaps of 256 / 1024 (shared
    memory) and 1025 (global memory) entries; each length includes frames of zeros once it is long enough"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    paths = ["default"]
    combos = [(t, r, L) for t in (False, True) for r in RANGES for L in CMAPS]
    k = 0
    for path in paths:
        for ov in OVERLAPS:
            hop = W - int(ov * W)
            ns = lengths(W, hop)
            for i, n in enumerate(ns):
                x = capture(n, W, seed=n)
                todo = combos if i == len(ns) - 1 else [combos[(k + d) % len(combos)] for d in range(3)]
                k += 3
                for transpose, (lo, hi), L in todo:
                    spec = Spectrogram(x, W, ov)
                    spec.data_min, spec.data_max = lo, hi
                    got = spec.create_spectrogram_image(transpose=transpose, colormap=CMAPS[L])
                    want = composed(spec, x, transpose, CMAPS[L])
                    assert got.shape == want.shape and got.dtype == np.uint8, (got.shape, want.shape)
                    bad = np.argwhere(np.any(got != want, axis=-1))
                    assert len(bad) == 0, (path, W, ov, n, transpose, lo, hi, L, bad[:8])


def test_all_zero_capture_is_entry_zero():
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    for W in (1024, 1000):
        x = np.zeros(5 * W, np.complex64)
        img = Spectrogram(x, W).create_spectrogram_image(colormap=CMAPS[256])
        assert img.shape == (W, 9, 4) and np.all(img == CMAPS[256][0])


def test_slices_and_device_samples(ctx):
    """numpy slice semantics (start / end / step, negative step) on host and device samples; a DeviceArray of complex64 or
    float32 (n, 2) gives the same image as the numpy capture"""
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    x = capture(40_000, 1024, seed=3)
    d_c = to_device(x, ctx)
    d_f = to_device(x.view(np.float32).reshape(-1, 2), ctx)
    for args in [(), (100, 9000), (None, 5000, 3), (30_000, 2000, -7), (5, 5), (39_000, None)]:
        for transpose in (False, True):
            want = Spectrogram(x[slice(*args)] if args else x).create_spectrogram_image(transpose=transpose, colormap=CMAPS[256])
            host = Spectrogram(x).create_spectrogram_image(*args, transpose=transpose, colormap=CMAPS[256])
            assert np.array_equal(host, want), args
            for d in (d_c, d_f):
                got = Spectrogram(d).create_spectrogram_image(*args, transpose=transpose, colormap=CMAPS[256])
                assert got.shape == want.shape and np.array_equal(got.get(), want), (args, transpose, d.dtype)


@pytest.mark.parametrize("W,ov,n", [(1024, 0.5, 2_000_000), (256, 0.75, 700_001), (1000, 0.5, 1_100_003), (128, 0, 300_000)])
def test_image_segments_one_launch(ctx, W, ov, n):
    """create_image_segments: the reference's slices (segment_bounds, pinned on the CPU), each image equal to
    create_spectrogram_image(start, start + step) bit for bit, one kernel launch for all of them on the fused path, and the same
    images from a DeviceArray"""
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    x = capture(n, W, seed=W)
    spec = Spectrogram(x, W, ov)
    bounds = spec.segment_bounds()
    assert len(bounds) > 1
    list(spec.create_image_segments(colormap=CMAPS[256]))   # twiddles of this W now cached
    before = ctx.launch_count()
    segs = list(spec.create_image_segments(colormap=CMAPS[256]))
    launches = ctx.launch_count() - before
    if (W & (W - 1)) == 0:
        assert launches == 1, launches
    assert len(segs) == len(bounds)
    step = bounds[0][1] - bounds[0][0]
    for (s, e, frames), img in zip(bounds, segs):
        assert img.shape == (W, frames, 4)
        assert np.array_equal(img, spec.create_spectrogram_image(s, s + step, colormap=CMAPS[256])), (s, e)
    dev = list(Spectrogram(to_device(x, ctx), W, ov).create_image_segments(colormap=CMAPS[256]))
    assert len(dev) == len(segs) and all(np.array_equal(d.get(), h) for d, h in zip(dev, segs))


# ---- against the reference's own Spectrogram ---------------------------------------------------------------------------------
def reference_layer():
    from oracle import ref_loader

    if not ref_loader.python_layer_available():
        pytest.skip("the reference's Python layer is not staged (oracle/_ref/pyref)")
    ns = ref_loader.load_python_layer()
    from urh import colormaps
    return ns, colormaps


def test_image_against_reference_composition():
    """The reference's create_spectrogram_image (its own float64 FFT, magma colormap) on the fixture of its test_spectrogram.py:
    same shape (width = time_bins - 2, height = freq_bins); the colormap index within +-1 of the reference's wherever the dB value is
    within 150 dB of its frame's peak, and identical wherever the reference's normalised value is more than (L-1) 1e-3 / (max - min)
    from an integer (1e-3 dB is the dB map's bar, DESIGN 4.6)"""
    from conftest import load_golden
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    ns, colormaps = reference_layer()
    cmap = colormaps.calculate_numpy_brga_for("magma")
    colormaps.chosen_colormap_numpy_bgra = cmap
    lut = {int(v): i for i, v in enumerate(cmap.view(np.uint32)[:, 0])}
    assert len(lut) == len(cmap)
    iq = load_golden("capture_two_participants")["iq"]
    for transpose in (False, True):
        for W, ov, (lo, hi) in [(1024, 0.5, (-140, 10)), (1024, 0.5, (-80, 10)), (256, 0.75, (-140, 10)), (1000, 0.3, (-140, 10))]:
            ref = ns.Spectrogram(iq, window_size=W, overlap_factor=ov)
            ref.data_min, ref.data_max = lo, hi
            want = ref.create_spectrogram_image(transpose=transpose).data
            spec = Spectrogram(iq, W, ov)
            spec.data_min, spec.data_max = lo, hi
            got = spec.create_spectrogram_image(transpose=transpose, colormap=cmap)
            assert got.shape == want.shape, (got.shape, want.shape)
            if not transpose and W == 1024 and ov == 0.5:
                assert (want.shape[1], want.shape[0]) == (ref.time_bins - 2, ref.freq_bins)
            db = ref._Spectrogram__calculate_spectrogram(ref.samples)
            data = np.flipud(db.T) if transpose else db
            norm = (len(cmap) - 1) * ((data.T - lo) / (hi - lo))   # what the reference truncates
            ref_idx = np.vectorize(lut.get)(want.view(np.uint32)[..., 0])
            got_idx = np.vectorize(lut.get)(got.view(np.uint32)[..., 0])
            peak = db.max(axis=1)   # per frame
            frame_peak = (peak[None, :] if not transpose else peak[:, None]) * np.ones(norm.shape)
            strong = data.T >= frame_peak - 150
            assert np.all(np.abs(got_idx - ref_idx)[strong] <= 1), (W, ov, transpose)
            with np.errstate(invalid="ignore"):
                far = np.abs(norm - np.round(norm)) > (len(cmap) - 1) * 1e-3 / (hi - lo)
            assert np.array_equal(got_idx[strong & far], ref_idx[strong & far]), (W, ov, transpose)


# ---- FTA export ---------------------------------------------------------------------------------------------------------------
def fta_captures():
    from conftest import load_golden

    out = {name: load_golden("capture_" + name)["iq"] for name in ("fsk", "ask", "enocean")}
    rng = np.random.default_rng(9)
    out["seeded"] = (rng.standard_normal((300_000, 2)) * 0.1).astype(np.float32)
    out["seeded"][100_000:103_000] = 0
    return out


@pytest.mark.parametrize("include_amplitude", [False, True])
def test_fta_export_equals_restatement(monkeypatch, tmp_path, include_amplitude):
    """the exported file == the restatement (tests/fta_restatement.py) applied to the device's own dB map, byte for byte; the
    seeded capture also with bands of a few rows (band constant made small), so that many bands alternate between the buffers"""
    from urh_b200.signalprocessing import Spectrogram as mod

    for name, iq in fta_captures().items():
        for band in ([None, 3 * 1024 * 48 + 5] if name == "seeded" else [None]):
            if band:
                monkeypatch.setattr(mod, "FTA_BAND_BYTES", band)
            spec = mod.Spectrogram(iq)
            path = tmp_path / ("%s_%s.fta" % (name, band))
            spec.export_to_fta(2e6, str(path), include_amplitude)
            want = fta_bytes(spec.calculate_spectrogram(), len(iq), 2e6, include_amplitude)
            got = path.read_bytes()
            assert len(got) == len(want) and got == want, (name, band)
            monkeypatch.setattr(mod, "FTA_BAND_BYTES", 64 << 20)


def test_fta_export_against_reference_file(tmp_path):
    """against the reference's own export_to_fta: f and t bytes identical, a within 1e-3 dB inside the 150 dB window of its frame,
    -inf in the same places"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    ns, _ = reference_layer()
    for name, iq in fta_captures().items():
        if name == "seeded":
            continue
        ref_path, path = tmp_path / (name + "_ref.fta"), tmp_path / (name + ".fta")
        ns.Spectrogram(iq).export_to_fta(1e6, str(ref_path), True)
        Spectrogram(iq).export_to_fta(1e6, str(path), True)
        dt = np.dtype([("f", np.float64), ("t", np.uint32), ("a", np.float32)])
        want, got = np.fromfile(str(ref_path), dt), np.fromfile(str(path), dt)
        assert len(want) == len(got)
        assert np.array_equal(want["f"].view(np.uint64), got["f"].view(np.uint64)), name
        assert np.array_equal(want["t"], got["t"]), name
        W = 1024
        a_ref, a = want["a"].reshape(W, -1, 3)[:, :, 0], got["a"].reshape(W, -1, 3)[:, :, 0]
        assert np.array_equal(np.isneginf(a_ref), np.isneginf(a)), name
        strong = a_ref >= a_ref.max(axis=0, keepdims=True) - 150
        assert np.all(np.abs(a - a_ref)[strong] <= 1e-3), (name, np.abs(a - a_ref)[strong].max())


def test_fta_export_overflow_creates_no_file(tmp_path):
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    x = capture(1 << 16, 1024)
    path = tmp_path / "big.fta"
    with pytest.raises(OverflowError, match="out of bounds for uint32"):
        Spectrogram(x).export_to_fta(10.0, str(path), True)
    assert not path.exists()
