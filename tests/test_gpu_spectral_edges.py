"""GPU: the named cases of tests/spectral_edge_cases.py through every device entry of the filter and spectrogram family, against the
oracle (pinned to the reference in tests/test_oracle.py).  The bars where a value is finite are tests/test_gpu_spectral.py's.
  STFT, dB map, FTA amplitudes: per-component classes equal the oracle's in every bin (a frame that reads a non-finite sample is
    NaN + NaN j, its dB values NaN); finite frames within 1e-12 of the frame peak (STFT) and 1e-3 dB within 150 dB (dB map).
  images: numpy's look-up of the device's dB map bit for bit, and of the oracle's dB map in every frame that reads a non-finite sample.
  band-pass, fft_convolve_1d: per-component classes equal the oracle's on both branches (the FFT branch: one non-finite sample makes
    every output NaN + NaN j), finite values within one float32 rounding of the float64 result and 1e-5 of the scale of the oracle's;
    the reference's single-precision transform overflowing on samples near FLT_MAX is the one documented difference.
  DC correction: word for word (NaN folded, -0 apart from +0) up to 2^22 float32 rows and for integers; above, x - float32(float64 mean)."""
import contextlib
import ctypes as C
import warnings

import numpy as np
import pytest

from spectral_edge_cases import EXACT_DC_MAX, answers, bad_frames, cases, classes, folded, hop_of, segment_bounds
from test_gpu_spectral import DB_ABS, DB_RANGE, STFT_REL
from test_gpu_stream_filters import low_budget  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

CASES = cases()
CMAP = np.random.default_rng(4).integers(0, 256, (256, 4)).astype(np.uint8)


@pytest.fixture(scope="module")
def ctx():
    from urh_b200 import _lib

    if not _lib.cuda_available():
        pytest.skip("no CUDA device")
    return _lib.default_context()


def _of(group):
    return [c for c in CASES if c.group in group]


def _quiet():
    """a context with numpy's floating-point warnings off (the cases form inf and NaN on purpose)"""
    stack = contextlib.ExitStack()
    stack.enter_context(warnings.catch_warnings())
    warnings.simplefilter("ignore", RuntimeWarning)
    stack.enter_context(np.errstate(all="ignore"))
    return stack


def oracle_answers(oracle, case):
    return dict(answers(case, stft=oracle.stft, spectrogram_db=lambda x, W, ov: oracle.spectrogram_db(x, W, ov),
                        fta=lambda x, W, ov: np.flipud(oracle.spectrogram_db(x, W, ov).T),
                        apply_bandpass_filter=oracle.apply_bandpass_filter, fft_convolve_1d=oracle.fft_convolve_1d,
                        dc_correction=oracle.dc_correction))


def check_stft(got, ref, bad, key):
    assert got.shape == ref.shape and got.dtype == np.complex128, (key, got.shape, ref.shape)
    assert np.array_equal(classes(got), classes(ref)), (key, np.argwhere(classes(got) != classes(ref))[:8])
    assert np.isnan(got[bad].real).all() and np.isnan(got[bad].imag).all(), key
    ok = ~bad
    peak = np.abs(ref[ok]).max(axis=1) if ok.any() else np.zeros(0)
    err = np.abs(got[ok] - ref[ok]).max(axis=1) if ok.any() else np.zeros(0)
    assert np.all(err <= STFT_REL * peak), (key, err, peak)


def check_db(got, ref, bad, key):
    """classes equal in every bin, except that -inf and a finite value below the frame's 150 dB floor are one class (an exact zero
    in one complex64 cast and a rounding residue in the other: test_gpu_spectral.check_db's rule)"""
    assert got.shape == ref.shape and got.dtype == np.float32, (key, got.shape, ref.shape)
    fin = np.isfinite(ref)
    peak = np.where(fin, ref, -np.inf).max(axis=1, keepdims=True)
    with np.errstate(invalid="ignore"):
        floor_g = np.isneginf(got) | (np.isfinite(got) & (got < peak - DB_RANGE))
        floor_r = np.isneginf(ref) | (fin & (ref < peak - DB_RANGE))
    cg, cr = np.where(floor_g, 4, classes(got)), np.where(floor_r, 4, classes(ref))
    assert np.array_equal(cg, cr), (key, np.argwhere(cg != cr)[:8])
    assert np.isnan(got[bad]).all(), key
    strong = fin & (ref >= peak - DB_RANGE)
    d = np.where(strong, np.abs(got.astype(np.float64) - ref), 0.0)
    assert np.all(d <= DB_ABS), (key, d.max())
    weak = fin & ~strong
    assert np.all(~weak | (got < peak - DB_RANGE + 1.0)), key


def lookup(db, lo=-140, hi=10):
    """Spectrogram.apply_bgra_lookup in numpy (the reference's expression)"""
    with np.errstate(all="ignore"):
        v = (len(CMAP) - 1) * ((db.T - lo) / (hi - lo))
        return np.take(CMAP, v.astype(int), axis=0, mode="clip")


# ---- STFT, dB map, FTA -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [64, 128, 1000, 1001, 1024, 4096])
def test_stft_db_fta_edges(ctx, oracle, W, tmp_path):
    """host arrays, DeviceArray samples and a view one sample into a device buffer; the FTA amplitudes of the small cases"""
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    w = _quiet()
    try:
        for case in [c for c in _of(("stft",)) if c.W == W]:
            ref = oracle_answers(oracle, case)
            hop = hop_of(W, case.ov)
            bad = bad_frames(case.x, W, hop)
            spec = Spectrogram(case.x, W, case.ov)
            check_stft(spec.stft(case.x), ref["stft"], bad, case.name)
            check_db(spec.calculate_spectrogram(), ref["db"], bad, case.name)
            if len(case.x):
                d = to_device(case.x.view(np.float32).reshape(-1, 2), ctx)
                check_stft(spec.stft(d), ref["stft"], bad, (case.name, "device"))
                buf = to_device(np.concatenate([np.zeros(1, np.complex64), case.x]).view(np.float32).reshape(-1, 2), ctx)
                view = DeviceArray(ctx, (len(case.x), 2), np.float32, buf.ptr + 8, base=buf)
                check_db(spec.calculate_spectrogram(view), ref["db"], bad, (case.name, "view"))
            if "fta" in ref:
                path = str(tmp_path / "x.fta")
                spec.export_to_fta(1e6, path, include_amplitude=True)
                a = np.fromfile(path, dtype=Spectrogram.fta_dtype(True))["a"].reshape(W, -1, 3)[:, :, 0]
                assert np.array_equal(classes(a), classes(ref["fta"])), case.name
                assert np.array_equal(folded(a), folded(np.flipud(spec.calculate_spectrogram().T))), case.name
    finally:
        w.__exit__(None, None, None)


def test_stft_hop_zero_raises_like_the_reference():
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    with pytest.raises(ZeroDivisionError):
        Spectrogram(np.ones(100, np.complex64), 64, 1.0).stft(np.ones(100, np.complex64))


@pytest.mark.parametrize("ring", [2, 3])
def test_stft_db_images_streamed(ctx, oracle, low_budget, monkeypatch, ring):  # noqa: F811
    """the windowed ring: a budget below the resident call, small chunks, the bad samples in later chunks and chunk halos"""
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    monkeypatch.setattr(sf, "STREAM_RING", ring)
    w = _quiet()
    try:
        for case in _of(("segments",)):
            ref = oracle_answers(oracle, case)
            hop = hop_of(case.W, case.ov)
            bad = bad_frames(case.x, case.W, hop)
            spec = Spectrogram(case.x, case.W, case.ov)
            resident_db = spec.calculate_spectrogram()
            resident_img = list(spec.create_image_segments(colormap=CMAP))
            low_budget()
            check_stft(spec.stft(case.x), ref["stft"], bad, (case.name, "stream"))
            db = spec.calculate_spectrogram()
            check_db(db, ref["db"], bad, (case.name, "stream"))
            assert np.array_equal(folded(db), folded(resident_db))
            imgs = list(spec.create_image_segments(colormap=CMAP))
            assert all(np.array_equal(a, b) for a, b in zip(imgs, resident_img)) and len(imgs) == len(resident_img)
            assert {"urh_stft_stream", "urh_spectrogram_db_stream", "urh_spectrogram_bgra_stream"} <= set(low_budget.streamed)
            monkeypatch.delenv("URH_B200_DEVICE_BUDGET")
    finally:
        w.__exit__(None, None, None)


# ---- images ----------------------------------------------------------------------------------------------------------------------------
def test_images_edges(ctx, oracle):
    """create_image_segments and create_spectrogram_image (both layouts) on captures with a non-finite sample on every segment
    boundary, and the per-rank segment windows of dist.segment_plan on one GPU"""
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    w = _quiet()
    try:
        for case in _of(("segments",)):
            W, hop = case.W, hop_of(case.W, case.ov)
            ref = oracle_answers(oracle, case)
            spec = Spectrogram(case.x, W, case.ov)
            bounds = segment_bounds(len(case.x), W, hop)
            assert [(s, e) for s, e, _ in spec.segment_bounds()] == bounds and len(bounds) >= 3
            imgs = list(spec.create_image_segments(colormap=CMAP))
            assert len(imgs) == len(bounds)
            read = 0
            for i, ((s, e), img) in enumerate(zip(bounds, imgs)):
                seg = case.x[s:e]
                bad = bad_frames(seg, W, hop)
                read += int(bad.any())
                own_db = Spectrogram(seg, W, case.ov).calculate_spectrogram()
                assert np.array_equal(img, lookup(own_db)), (case.name, i)
                want = lookup(ref["db_seg%d" % i])
                assert np.array_equal(img[:, bad], want[:, bad]), (case.name, i)
                t = spec.create_spectrogram_image(s, e, transpose=True, colormap=CMAP)
                assert np.array_equal(t, lookup(np.flipud(own_db.T))), (case.name, i)
            assert read >= len(bounds) - 1, (case.name, read)   # the first segment's last sample may lie past its last frame
            n = len(case.x)
            shards = [(0, n // 3 + 5), (n // 3 + 5, 2 * n // 3 + 1), (2 * n // 3 + 1, n)]
            segs, owned, rights = udist.segment_plan(n, W, hop, shards)
            for (g0, g1), mine, right in zip(shards, owned, rights):
                local = Spectrogram(case.x[g0: g1 + right], W, case.ov)
                for i in mine:
                    s, e, _ = segs[i]
                    assert np.array_equal(local.create_spectrogram_image(s - g0, e - g0, colormap=CMAP), imgs[i]), (case.name, i)
    finally:
        w.__exit__(None, None, None)


def test_db_map_per_rank_frames(ctx, oracle):
    """dist.frame_plan's per-rank windows through urh_spectrogram_db on one GPU: the whole capture's dB map, NaN frames included"""
    from urh_b200 import dist as udist
    from urh_b200.device import DeviceArray, to_device

    w = _quiet()
    try:
        for case in _of(("segments",)):
            W, hop, n = case.W, hop_of(case.W, case.ov), len(case.x)
            ref = oracle_answers(oracle, case)["db"]
            d_w = to_device(np.hanning(W).astype(np.float64), ctx)
            bounds = [(0, n // 3 + 7), (n // 3 + 7, n // 2 + 1), (n // 2 + 1, n)]
            rows = []
            for (g0, g1), (f0, nf, right) in zip(bounds, udist.frame_plan(n, W, hop, bounds)):
                if nf:
                    win = np.ascontiguousarray(case.x[f0 * hop: g1 + right])
                    d_x = to_device(win.view(np.float32), ctx)
                    out = DeviceArray(ctx, (nf, W), np.float32)
                    ctx.check(ctx.lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr), len(win), W, hop, C.c_void_p(d_w.ptr), nf,
                                                         C.c_void_p(out.ptr)))
                    rows.append(out.get())
            check_db(np.concatenate(rows), ref, bad_frames(case.x, W, hop), case.name)
    finally:
        w.__exit__(None, None, None)


# ---- band-pass and fft_convolve_1d -----------------------------------------------------------------------------------------------------
def _fft_overflow(case, fft_branch):
    """the reference's single-precision transform of a complex64 capture overflows on samples near FLT_MAX (DESIGN.md §4.5)"""
    return fft_branch and ("fft_overflow" in case.name or "huge_3e38" in case.name)


def check_filter(got, case, oracle, fft_branch, key):
    ref = oracle_answers(oracle, case)["out"]
    exact = (oracle.apply_bandpass_filter(case.x.astype(np.complex128), case.f_low, case.f_high, case.bw) if case.group == "bandpass"
             # the shim takes the samples as complex64: the float64 result of the same operation is that of the rounded samples
             else oracle.fft_convolve_1d(case.x.astype(np.complex64).astype(np.complex128) if np.iscomplexobj(case.x)
                                         else case.x.astype(np.float32).astype(np.float64),
                                         np.asarray(case.h, dtype=np.complex128 if np.iscomplexobj(case.h) else np.float64)))
    assert got.shape == ref.shape, (key, got.shape, ref.shape)
    if case.group == "convolve":
        assert got.dtype == (ref.dtype if ref.dtype != np.complex128 else np.complex64), (key, got.dtype, ref.dtype)
    if _fft_overflow(case, fft_branch):
        assert np.isnan(ref).all() and np.isfinite(exact).all() and np.isfinite(got).all(), key
    elif fft_branch:
        assert np.array_equal(classes(got), classes(ref)), (key, np.argwhere(classes(got) != classes(ref))[:8])
    else:
        # np.convolve's complex dot product may pair the infinite partial products of one output differently (NaN where the kernel's
        # per-term sum keeps +-inf in a part): the outputs that are not finite are the same ones
        assert np.array_equal(np.isfinite(got), np.isfinite(ref)), (key, np.argwhere(np.isfinite(got) != np.isfinite(ref))[:8])
    fin = np.isfinite(exact) & np.isfinite(got)
    if fin.any():
        g, r = got[fin].astype(np.complex128), exact[fin].astype(np.complex128)
        scale = np.abs(r).max()
        for part in (np.real, np.imag):
            # one float32 rounding (2^-150 absolute below FLT_MIN) + 1e-12 of the scale (test_gpu_spectral.check_conv)
            bar = 2.0 ** -24 * np.abs(part(r)) * (1 + 1e-6) + 1e-12 * scale + 2.0 ** -150
            assert np.all(np.abs(part(g) - part(r)) <= bar), (key, np.argwhere(np.abs(part(g) - part(r)) > bar)[:8])
        # against the reference's own single-precision transform, where its scale is normal
        if np.isfinite(ref[fin]).all() and np.abs(ref[fin]).max() >= 1e-30:
            assert np.abs(g - ref[fin]).max() <= 1e-5 * np.abs(ref[fin]).max(), key


def _bandpass_branch(case):
    from urh_b200.signalprocessing.Filter import Filter

    m = len(Filter.bandpass_taps(case.f_low, case.f_high, case.bw))
    return not m < 8 * np.log(np.sqrt(len(case.x)))


def test_bandpass_and_convolve_edges(ctx, oracle):
    from urh_b200.signalprocessing.Filter import Filter

    w = _quiet()
    try:
        for case in _of(("bandpass",)):
            check_filter(Filter.apply_bandpass_filter(case.x, case.f_low, case.f_high, case.bw), case, oracle, _bandpass_branch(case),
                         case.name)
        for case in _of(("convolve",)):
            check_filter(Filter.fft_convolve_1d(case.x, case.h), case, oracle, True, case.name)
    finally:
        w.__exit__(None, None, None)


@pytest.mark.parametrize("ring", [2, 3])
def test_bandpass_streamed(ctx, oracle, low_budget, monkeypatch, ring):  # noqa: F811
    """urh_convolve_c128_stream with chunks of 2^14 samples: the bad sample lands in a later chunk or a halo"""
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Filter import Filter

    monkeypatch.setattr(sf, "STREAM_RING", ring)
    low_budget()
    w = _quiet()
    try:
        for case in _of(("bandpass",)):
            if "huge" in case.name or "subnormal" in case.name:
                continue
            before = dict(low_budget.streamed)
            got = Filter.apply_bandpass_filter(case.x, case.f_low, case.f_high, case.bw)
            assert low_budget.streamed != before, case.name
            check_filter(got, case, oracle, _bandpass_branch(case), (case.name, "stream", ring))
        # a capture of many chunks with one non-finite sample in a halo between two chunks, FFT branch (401 taps)
        n = 5 * (1 << 14) + 333
        x = (np.random.default_rng(ring).standard_normal(n) * (1 + 0j)).astype(np.complex64)
        x[3 * (1 << 14) + 100] = np.inf
        y = Filter.apply_bandpass_filter(x, 0.1, 0.2, 0.01)
        assert np.isnan(y.real).all() and np.isnan(y.imag).all()
    finally:
        w.__exit__(None, None, None)


def test_bandpass_per_rank_windows(ctx, oracle):
    """dist.bandpass_plan's windows on one GPU, with the rule dist.apply_bandpass_filter_sharded applies on the FFT branch: each rank
    flags its own outputs (urh_nonfinite_flag), the flags are OR-ed over the ranks, and every rank fills its output (urh_nan_fill_if)"""
    from urh_b200 import dist as udist
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Filter import Filter

    w = _quiet()
    try:
        for case in _of(("bandpass",)):
            n = len(case.x)
            if n < 10_000:
                continue
            h = np.ascontiguousarray(Filter.bandpass_taps(case.f_low, case.f_high, case.bw), dtype=np.complex128)
            fft_branch = _bandpass_branch(case)
            bounds = [(0, 1280 * 3 + 1), (1280 * 3 + 1, n // 2), (n // 2, n)]
            d_t = to_device(h.view(np.float64), ctx)
            outs, flags = [], []
            for (g0, g1), (left, right, offset) in zip(bounds, udist.bandpass_plan(n, len(h), bounds)):
                d_x = to_device(np.ascontiguousarray(case.x[g0 - left: g1 + right]).view(np.float32), ctx)
                out = DeviceArray(ctx, (g1 - g0,), np.complex64)
                ctx.check(ctx.lib.urh_convolve_c128(ctx.handle, C.c_void_p(d_x.ptr), left + g1 - g0 + right, C.c_void_p(d_t.ptr), len(h),
                                                    int(offset), g1 - g0, C.c_void_p(out.ptr)))
                flag = to_device(np.zeros(1, np.int32), ctx)
                ctx.check(ctx.lib.urh_nonfinite_flag(ctx.handle, C.c_void_p(out.ptr), g1 - g0, C.c_void_p(flag.ptr)))
                outs.append(out)
                flags.append(int(flag.get()[0]))
            if fft_branch and any(flags):
                one = to_device(np.ones(1, np.int32), ctx)
                for out in outs:
                    ctx.check(ctx.lib.urh_nan_fill_if(ctx.handle, C.c_void_p(out.ptr), len(out), C.c_void_p(one.ptr)))
            got = np.concatenate([o.get() for o in outs])
            assert np.array_equal(folded(got), folded(Filter.apply_bandpass_filter(case.x, case.f_low, case.f_high, case.bw))), case.name
            check_filter(got, case, oracle, fft_branch, (case.name, "ranks"))
    finally:
        w.__exit__(None, None, None)


# ---- DC correction ---------------------------------------------------------------------------------------------------------------------
def check_dc(got, case, oracle, key):
    x = case.x
    assert got.dtype == (np.float32 if x.dtype == np.float32 else np.float64) and got.shape == x.shape, key
    if x.dtype != np.float32 or len(x) <= EXACT_DC_MAX:
        assert np.array_equal(folded(got), folded(oracle.dc_correction(x))), key
        return
    m32 = np.mean(x.astype(np.float64), axis=0).astype(np.float32)
    assert np.array_equal(folded(got), folded(x - m32)), key
    if "overflow" in case.name:   # the float32 sums overflow, the double sums do not
        assert not np.isfinite(oracle.dc_correction(x)[:, 0]).any() and np.isfinite(got[:, 0]).any(), key


def test_dc_correction_edges(ctx, oracle):
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Filter import Filter, FilterType

    w = _quiet()
    try:
        for case in _of(("dc",)):
            check_dc(Filter.dc_correction(case.x), case, oracle, case.name)
            check_dc(Filter([], FilterType.dc_correction).work(case.x), case, oracle, (case.name, "work"))
            if case.x.dtype == np.float32:
                # the per-rank split: serial chain handed over in row order (<= 2^22 rows) or double sums folded in rank order
                n = len(case.x)
                d = to_device(case.x, ctx)
                cuts = [(0, n // 3), (n // 3, n)] if n >= 3 else [(0, n)]
                exact = int(n <= EXACT_DC_MAX)
                carry, dsum = np.zeros(2, np.float32), np.zeros(2, np.float64)
                for a, b in cuts:
                    s = np.zeros(2, np.float64)
                    ctx.check(ctx.lib.urh_dc_column_sums(ctx.handle, C.c_void_p(d[a:b].ptr), b - a, exact,
                                                         carry.ctypes.data_as(C.c_void_p) if exact else None, s.ctypes.data_as(C.c_void_p)))
                    carry, dsum = s.astype(np.float32), dsum + s
                mean = carry / np.float32(n) if exact else (dsum / n).astype(np.float32)
                check_dc(case.x - mean, case, oracle, (case.name, "split"))
    finally:
        w.__exit__(None, None, None)


@pytest.mark.parametrize("ring", [2, 3])
def test_dc_correction_streamed(ctx, oracle, low_budget, monkeypatch, ring):  # noqa: F811
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.signalprocessing.Filter import Filter

    monkeypatch.setattr(sf, "STREAM_RING", ring)
    low_budget()
    w = _quiet()
    try:
        for case in _of(("dc",)):
            if len(case.x) < 1 << 16:
                continue
            before = dict(low_budget.streamed)
            check_dc(Filter.dc_correction(case.x), case, oracle, (case.name, "stream", ring))
            assert low_budget.streamed != before, case.name
    finally:
        w.__exit__(None, None, None)
