"""GPU: every kernel path of spectrogram.cu and filter.cu that the run-time dispatch can select, against float64 references of
the same operation (oracle/oracle.py, numpy), at the sizes where the dispatch switches and the kernels' tiles end.

Paths (DESIGN 4.5 / 4.6):
  STFT     powers of two 128 .. 4096: k_stft_r16 (radix-16 passes + one radix-2 / 4 / 8 pass);
           everything else: k_stft_window -> cuFFT Z2Z -> k_stft_scale / k_stft_db, in 512 MiB batches
  band-pass  m <= 768 taps: k_conv_c128_tiled;  more: k_conv_c128
  DC       n <= Filter.EXACT_DC_MAX: k_dc_mean_serial (numpy's float32 chain);  more: k_dc_mean_partial + k_dc_mean_fold (double)

Run with -s to see the largest error each path showed (the STFT and dB map per window size)."""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

STFT_SIZES = [64, 128, 256, 512, 1000, 1001, 1024, 2048, 3000, 4096, 8192]
OVERLAPS = [0, 0.5, 0.75, 0.3]
STFT_REL = 1e-12    # per frame: max|got - ref| <= STFT_REL * max|ref frame|   (a double FFT is ~1e-15; float twiddles ~3e-8)
DB_ABS = 1e-3       # dB, in every bin within DB_RANGE of its frame's peak (DESIGN 4.6)
DB_RANGE = 150.0

WORST = {}          # path -> largest error seen, printed at the end of the module


def _record(key, value):
    WORST[key] = max(WORST.get(key, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(WORST):
        print("%-48s %.6g" % (key, WORST[key]))


def asymmetric(w):
    """seeded values in (0.5, 1]: unlike np.hanning, a window applied back to front gives a different transform"""
    return 1.0 - 0.5 * np.random.default_rng(w).random(w)


WINDOWS = {"hanning": np.hanning, "asymmetric": asymmetric}


def stft_kernel(W):
    return "k_stft_r16" if (W & (W - 1)) == 0 and 128 <= W <= 4096 else "cufft"


def lengths(W, hop):
    """0, 1, one short of / exactly / one past a frame, one short of / exactly a second frame, ~20 frames and a partial one"""
    return sorted({0, 1, W - 1, W, W + 1, W + hop - 1, W + hop, W + 20 * hop + hop // 2})


def capture(n, W, seed=1):
    """DC offset + a strong tone; the first half without noise (Hanning sidelobes of a clean tone reach far below the peak:
    weak bins), then noise, interrupted by 2 W exact zeros (whole frames of zeros once there are enough frames)"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = (0.25 - 0.5j) + 2.0 * np.exp(2j * np.pi * 0.1937 * t)
    x[n // 2:] += 1e-3 * (rng.standard_normal(n - n // 2) + 1j * rng.standard_normal(n - n // 2))
    x[n // 2 + W // 2: n // 2 + W // 2 + 2 * W] = 0
    return x.astype(np.complex64)


def check_stft(got, ref, key):
    assert got.shape == ref.shape and got.dtype == np.complex128, (got.shape, ref.shape, got.dtype)
    peak = np.abs(ref).max(axis=1)
    err = np.abs(got - ref).max(axis=1)
    # a frame of zeros must come out as exact zeros (bar 0)
    bad = np.nonzero(err > STFT_REL * peak)[0]
    assert len(bad) == 0, (key, "frames", bad[:8], err[bad[:8]], peak[bad[:8]])
    nz = peak > 0
    if nz.any():
        _record("stft rel err  %s W=%d" % key[:2], (err[nz] / peak[nz]).max())


def check_db(got, ref, key):
    """DESIGN 4.6 per frame: |delta| <= DB_ABS in every bin within DB_RANGE dB of the frame's peak; below that floor both sides
    stay below floor + 1 dB or are -inf; -inf in the reference (an exact complex64 zero) is -inf or below the floor here;
    a frame of zeros is -inf everywhere on both sides"""
    assert got.shape == ref.shape and got.dtype == np.float32, (got.shape, ref.shape, got.dtype)
    peak = ref.max(axis=1, keepdims=True)
    zero = np.isneginf(peak[:, 0])
    assert np.all(np.isneginf(got[zero])), (key, "zero frames", np.nonzero(zero)[0][:8])
    g, r, floor = got[~zero], ref[~zero], peak[~zero] - DB_RANGE
    strong = r >= floor
    with np.errstate(invalid="ignore"):
        d = np.where(strong, np.abs(g - r), 0.0)
    assert np.all(d <= DB_ABS), (key, "max |delta| dB", np.nanmax(d), np.argwhere(~(d <= DB_ABS))[:8])
    weak_ok = (g < floor + 1.0) | np.isneginf(g)
    assert np.all(weak_ok | strong), (key, "weak bins above floor + 1 dB", np.argwhere(~(weak_ok | strong))[:8])
    inf_ok = np.isneginf(g) | (g < floor)
    assert np.all(inf_ok | ~np.isneginf(r)), (key, "-inf in the reference", np.argwhere(~(inf_ok | ~np.isneginf(r)))[:8])
    if strong.any():
        _record("dB |delta|    %s W=%d" % key[:2], d.max())


# ---- 1. STFT (complex128) ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", sorted(WINDOWS))
@pytest.mark.parametrize("W", STFT_SIZES)
def test_stft_matches_float64_reference(oracle, W, window):
    """Spectrogram.stft on the kernel that serves W == oracle.stft (complex128, not rounded) to STFT_REL per frame"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    wf = WINDOWS[window]
    for ov in OVERLAPS:
        hop = W - int(ov * W)
        for n in lengths(W, hop):
            x = capture(n, W)
            ref = oracle.stft(x, W, ov, wf)
            check_stft(Spectrogram(x, W, ov, wf).stft(x), ref, (stft_kernel(W), W, ov, n, window))


# ---- 2. dB map (float32) -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", sorted(WINDOWS))
@pytest.mark.parametrize("W", STFT_SIZES)
def test_spectrogram_db_matches_float64_reference(oracle, W, window):
    """Spectrogram.calculate_spectrogram (fftshift, complex64 cast, dB, fliplr) on the kernel that serves W == oracle.spectrogram_db
    (check_db); odd W on cuFFT exercises k_stft_db's fftshift, the only place where it differs from W / 2"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    wf = WINDOWS[window]
    for ov in OVERLAPS:
        hop = W - int(ov * W)
        for n in lengths(W, hop):
            x = capture(n, W)
            ref = oracle.spectrogram_db(x, W, ov, window_function=wf)
            check_db(Spectrogram(x, W, ov, wf).calculate_spectrogram(), ref, (stft_kernel(W), W, ov, n, window))
        zeros = np.zeros(W + 5 * hop, np.complex64)
        ref = oracle.spectrogram_db(zeros, W, ov, window_function=wf)
        assert np.all(np.isneginf(ref))
        got = Spectrogram(zeros, W, ov, wf).calculate_spectrogram()
        assert got.shape == ref.shape and np.all(np.isneginf(got)), (W, ov)


# ---- 3. cuFFT batching and the plan cache ------------------------------------------------------------------------------------
def frame_db(oracle, x, W, hop, f, window):
    """row f of oracle.spectrogram_db, from that frame alone"""
    X = np.fft.fft(x[f * hop: f * hop + W] * window) / W
    return np.fliplr(oracle.arr2decibel(np.fft.fftshift(X)[None].astype(np.complex64)))


def test_spectrogram_cufft_batches_and_plan_cache(oracle):
    """W = 5000 (cuFFT), hop 2500: 6710 frames fill one 512 MiB batch, 6717 frames leave a last batch of 7 (ensure_plan rebuilds
    the plan).  Frames on either side of the batch boundary match the reference; a call of the last batch's 7 frames reuses the
    cached plan and repeats them bit for bit; after a call of another frame count rebuilt the plan, so does the first call"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    W, ov = 5000, 0.5
    hop = W - int(ov * W)
    max_batch = (512 << 20) // (W * 16)
    assert max_batch == 6710
    frames = max_batch + 7
    rng = np.random.default_rng(21)
    n = W + (frames - 1) * hop + 1234   # + a partial frame
    t = np.arange(n, dtype=np.float64)
    x = (np.exp(2j * np.pi * (0.05 + 0.2 * t / n) * t) + 1e-3 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    del t
    window = np.hanning(W)
    spec = Spectrogram(x, W, ov)
    first = spec.calculate_spectrogram(x)
    assert first.shape == (frames, W)
    for f in (0, max_batch - 1, max_batch, max_batch + 1, frames - 1):
        check_db(first[f:f + 1], frame_db(oracle, x, W, hop, f, window), ("cufft batched", W, f))
    tail = spec.calculate_spectrogram(x[max_batch * hop: max_batch * hop + W + 6 * hop])   # the last batch's frames, same plan
    assert tail.shape == (7, W) and bits_equal(tail, first[max_batch:]) == 0
    other = spec.calculate_spectrogram(x[: W + 99 * hop])   # 100 frames: plan rebuilt
    assert other.shape == (100, W)
    for f in (0, 99):
        check_db(other[f:f + 1], frame_db(oracle, x, W, hop, f, window), ("cufft batched", W, f))
    again = spec.calculate_spectrogram(x)
    assert bits_equal(again, first) == 0


# ---- 4. band-pass and urh_convolve_c128 -------------------------------------------------------------------------------------
def check_conv(got, ref, key):
    """per element and component: |got - ref| <= 2^-24 |ref| (1 + 1e-6)  (one rounding to float32)  +  1e-12 max|ref|
    (~1000 x the noise of a double accumulation)"""
    assert got.dtype == np.complex64 and got.shape == ref.shape, (got.dtype, got.shape, ref.shape)
    if ref.size == 0:
        return
    scale = np.abs(ref).max()
    g = got.astype(np.complex128)
    for part in (np.real, np.imag):
        r = part(ref)
        err = np.abs(part(g) - r)
        bar = 2.0 ** -24 * np.abs(r) * (1 + 1e-6) + 1e-12 * scale
        bad = np.nonzero(err > bar)[0]
        assert len(bad) == 0, (key, "elements", bad[:8], err[bad[:8]], bar[bad[:8]])
        # what the one rounding does not explain, against the 1e-12 term; and the error in float32 ulps where |ref| is not tiny
        _record("conv excess / max|ref|  " + key[0], ((err - 2.0 ** -24 * np.abs(r)) / scale).max())
        big = np.abs(r) >= 1e-3 * scale
        if big.any():
            ulp = np.spacing(np.abs(r[big]).astype(np.float32)).astype(np.float64)
            _record("conv err / float32 ulp  " + key[0], (err[big] / ulp).max())


def conv_kernel(m):
    return "k_conv_c128_tiled" if m <= 768 else "k_conv_c128"


def noise(rng, n):
    return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)


@pytest.mark.parametrize("n", [300, 5000, 1_500_000])
def test_bandpass_matches_float64_reference(oracle, n):
    """Filter.apply_bandpass_filter == oracle.apply_bandpass_filter (np.convolve 'same' / complex128 FFT) for every BANDWIDTHS
    preset (0.001 -> 4001 taps: untiled kernel).  At 1.5 M samples 11 / 41 / 51 taps take the direct branch and 401 / 4001 the
    FFT crop; both run past the first grid pass (~1.35 M outputs)"""
    from urh_b200.signalprocessing.Filter import Filter

    rng = np.random.default_rng(n)
    t = np.arange(n)
    x = (0.3 * noise(rng, n) + np.exp(2j * np.pi * 0.05 * t) + 0.5 * np.exp(-2j * np.pi * 0.4 * t)).astype(np.complex64)
    # numpy >= 2 transforms a complex64 array in single precision, so the reference's FFT branch is only ~3e-8 of the peak
    # accurate on complex64 input; the same samples as complex128 give the float64 result of the same operation
    x128 = x.astype(np.complex128)
    for name, bw in sorted(Filter.BANDWIDTHS.items()):
        m = Filter.get_filter_length_from_bandwidth(bw)
        for lo, hi in ((0.03, 0.07), (0.07, 0.03), (0.3, 0.9), (-0.9, -0.3)):
            ref = oracle.apply_bandpass_filter(x128, lo, hi, bw)
            got = Filter.apply_bandpass_filter(x, lo, hi, bw)
            check_conv(got, ref, (conv_kernel(m), name, m, n, lo, hi))


@pytest.mark.parametrize("m", [1, 2, 767, 768, 769, 4001])
def test_convolve_full_slice_matches_numpy(m):
    """Filter._convolve_full_slice == np.convolve(x, h, 'full')[offset : offset + out_len] in complex128 (zeros past n + m - 1):
    both kernels (the switch is 768 / 769 taps), from the start, from m - 1, running off the end, n < m, out_len % 1280 != 0"""
    from urh_b200.signalprocessing.Filter import Filter

    rng = np.random.default_rng(m)
    h = rng.standard_normal(m) + 1j * rng.standard_normal(m)
    for n in (19_999, 300):
        x = noise(rng, n)
        full = np.convolve(x.astype(np.complex128), h, "full")
        cases = [(0, n + m - 1), (m - 1, n), (max(n - 7, 0), m + 1500), (5, 2 * 1280 + 3)]
        assert any(out_len % 1280 for _, out_len in cases)
        for offset, out_len in cases:
            ref = np.zeros(out_len, np.complex128)
            seg = full[offset: offset + out_len]
            ref[: len(seg)] = seg
            got = Filter._convolve_full_slice(x, h, offset, out_len)
            check_conv(got, ref, (conv_kernel(m), m, n, offset, out_len))
            if offset + out_len > n + m - 1:
                assert np.all(got[n + m - 1 - offset:] == 0), (m, n, offset, out_len)


# ---- 5. DC correction --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2049, 1 << 22, (1 << 22) + 1, 5_000_000])
def test_dc_correction_both_paths(n):
    """n <= 2^22: numpy's own x - np.mean(x, axis=0) bit for bit (the serial float32 column sums; 1024 rows are one
    double-buffer chunk of k_dc_mean_serial).  n > 2^22: x - float32(the float64 mean) bit for bit, and visibly not numpy's"""
    from urh_b200.signalprocessing.Filter import Filter

    rng = np.random.default_rng(11)
    x = np.empty((n, 2), np.float32)
    x[:, 0] = 100 + rng.standard_normal(n)   # large offsets: the float32 chain drifts by percent at millions of rows
    x[:, 1] = -3 + rng.standard_normal(n)
    got = Filter.dc_correction(x)
    numpy_serial = x - np.mean(x, axis=0)
    if n <= Filter.EXACT_DC_MAX:
        assert bits_equal(got, numpy_serial) == 0
        return
    m64 = np.mean(x.astype(np.float64), axis=0)
    m32 = m64.astype(np.float32)
    # the device sums in another order than numpy; they round to the same float32 unless m64 sits on a rounding midpoint.
    # With this seed it is far from one (the smallest distance is ~3e-9 relative), so the comparison below is exact.
    for v, f in zip(m64, m32):
        mids = [(float(f) + float(np.nextafter(f, np.float32(s)))) / 2 for s in (-np.inf, np.inf)]
        assert min(abs(v - mid) for mid in mids) > 1e-9 * abs(v), (n, v)
    double_ref = x - m32
    assert bits_equal(got, double_ref) == 0
    assert bits_equal(double_ref, numpy_serial) > 0   # the two paths are told apart at this n
