"""Named, seeded inputs at the edges of the filter and spectrogram family: the band-pass and fft_convolve_1d (Filter.py:69-101), the
DC correction (Filter.py:31-33), the STFT, its dB map, the images and the FTA amplitudes (Spectrogram.py:94-190).

tests/test_oracle.py pins the oracle to the reference's own functions on them (recorded in tests/golden/ref_spectral_edges.json);
tests/test_gpu_spectral_edges.py runs them through every device entry against the oracle.  The groups:
* stft: W = 64, 1000, 1001 (cuFFT) and 128, 1024, 4096 (k_stft_r16), overlaps 0, 0.5 and 0.75, n = 0, 1, W - 1 and a few frames;
  +-inf, (inf, inf), (0, inf), NaN in either part at the first and last sample, a sample two frames read, a frame's first and last
  sample (np.hanning is exactly 0 there: inf * 0 is formed), inside the zero padding of n < W and in the last frame; huge values
  (1e30, 3.4e38, and samples whose float32 |X|^2 overflows), subnormals, signed zeros, all-zero and constant captures;
* segments: captures of several create_image_segments segments with a non-finite sample on each segment boundary;
* bandpass: the 41- and 51-tap presets on both sides of the 8 ln sqrt(n) branch switch, non-finite samples at 0, the last sample,
  within m - 1 of either end and at the edges of the 1280-output tile (CONV_TILE), huge, subnormal and signed-zero samples;
* convolve: fft_convolve_1d with 767 .. 769 taps, real x and real h (the reference's rfft branch returns float64), non-finite taps;
* dc: 1, 2, 1023, 1024, 1025, 2^22 and 2^22 + 1 rows; NaN in one column, +inf and -inf in one column, column sums that overflow
  float32, subnormal-only and -0.0-only columns, and the extremes of int8, uint8, int16 and uint16."""
import math

import numpy as np

C64 = np.complex64
INF, NAN = float("inf"), float("nan")
CONV_TILE = 1280
EXACT_DC_MAX = 1 << 22

# (real, imaginary) of every non-finite sample kind
NONFINITE = [(INF, 0.0), (-INF, 0.0), (INF, INF), (0.0, INF), (NAN, 0.0), (0.0, NAN)]
STFT_W = [64, 128, 1000, 1001, 1024, 4096]
OVERLAPS = [0, 0.5, 0.75]


class Case:
    __slots__ = ("name", "group", "x", "params")

    def __init__(self, name, group, x, **params):
        self.name, self.group, self.x, self.params = name, group, x, params

    def __getattr__(self, key):
        try:
            return self.params[key]
        except KeyError:
            raise AttributeError(key)


def c64(pairs):
    """a complex64 array of (re, im) pairs taken word for word (complex() would turn inf * 1j into nan + inf j)"""
    return np.ascontiguousarray(np.array(pairs, dtype=np.float32).reshape(-1, 2)).view(C64).ravel()


def noise(n, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * scale).astype(C64)


def classes(a):
    """per-component class of a real or complex array: 0 finite, 1 NaN, 2 +inf, 3 -inf (complex: trailing axis of 2, re and im)"""
    a = np.asarray(a)
    f = np.stack([a.real, a.imag], -1) if np.iscomplexobj(a) else a
    return np.select([np.isnan(f), np.isposinf(f), np.isneginf(f)], [1, 2, 3], 0).astype(np.uint8)


def folded(a):
    """the words of a result with every NaN folded to one NaN (the payload is not pinned); -0 and +0 stay apart"""
    a = np.asarray(a)
    f = np.stack([a.real, a.imag], -1) if np.iscomplexobj(a) else a
    w = np.ascontiguousarray(f).view(np.uint64 if f.dtype.itemsize == 8 else np.uint32).copy()
    w[np.isnan(f)] = 0x7FF8000000000000 if f.dtype.itemsize == 8 else 0x7FC00000
    return w


def hop_of(W, ov):
    return W - int(ov * W)


def frames_of(n, W, hop):
    return max(1, (max(n, W) - W) // hop + 1)


def bad_frames(x, W, hop):
    """bool per frame of Spectrogram.stft: does the frame read a non-finite sample"""
    n = len(x)
    bad = ~(np.isfinite(x.real) & np.isfinite(x.imag))
    F = frames_of(n, W, hop)
    pos = np.nonzero(bad)[0]
    out = np.zeros(F, bool)
    for p in pos:
        lo = max(0, -(-(p - W + 1) // hop))
        out[lo: min(F - 1, p // hop) + 1] = True
    return out


def branch_switch(m):
    """the least n for which Filter.apply_bandpass_filter with an m-tap filter takes np.convolve (m < 8 ln sqrt(n)) instead of the
    FFT convolution"""
    n = int(math.exp(m / 4.0)) - 2
    while not m < 8 * math.log(math.sqrt(n)):
        n += 1
    return n


def cases():
    with np.errstate(over="ignore", invalid="ignore"):
        return _cases()


def _cases():
    out = []

    def add(name, group, x, **params):
        out.append(Case(name, group, x, **params))

    # ---- STFT, dB map, images, FTA ------------------------------------------------------------------------------------------------
    for W in STFT_W:
        for ov in OVERLAPS:
            hop = hop_of(W, ov)
            key = "W%d_ov%g" % (W, ov)
            n = W + 4 * hop + hop // 2
            where = {"first": 0, "last": n - 1, "frame_first": 2 * hop, "frame0_last": W - 1,
                     "two_frames": hop + W // 3 if ov else W + W // 3, "last_frame": 4 * hop + W // 3}
            for i, (pos, p) in enumerate(where.items()):
                for j in (i % len(NONFINITE), (i + 3) % len(NONFINITE)):
                    x = noise(n, W + 7 * j + i)
                    x[p] = c64([NONFINITE[j]])[0]
                    add("stft_%s_%s_v%d" % (key, pos, j), "stft", x, W=W, ov=ov)
            for m, short in enumerate((1, W // 2, W - 1)):
                x = noise(short, W + short)
                x[short // 2] = c64([NONFINITE[(m + W) % len(NONFINITE)]])[0]
                add("stft_%s_padded_n%d" % (key, short), "stft", x, W=W, ov=ov)
            add("stft_%s_empty" % key, "stft", np.zeros(0, C64), W=W, ov=ov)
            add("stft_%s_zeros" % key, "stft", np.zeros(n, C64), W=W, ov=ov)
            add("stft_%s_constant" % key, "stft", np.full(n, 0.75 - 0.25j, C64), W=W, ov=ov)
            if ov == 0.5:
                add("stft_%s_huge_1e30" % key, "stft", noise(n, 3, 1e30), W=W, ov=ov)
                x = noise(n, 4)
                x[[1, W // 2]] = c64([(3.4e38, 0.0), (0.0, -3.4e38)])
                add("stft_%s_huge_3e38" % key, "stft", x, W=W, ov=ov)
                add("stft_%s_sq_overflow" % key, "stft", np.full(n, 4e19 + 4e19j, C64), W=W, ov=ov)   # float32 |X|^2 overflows
                add("stft_%s_subnormal" % key, "stft", np.tile(c64([(1e-45, 1e-40), (-1e-40, 1e-45)]), n // 2 + 1)[:n], W=W, ov=ov)
                add("stft_%s_neg_zero" % key, "stft", np.tile(c64([(0.0, -0.0), (-0.0, -0.0)]), n // 2 + 1)[:n], W=W, ov=ov)

    # ---- image segments: a non-finite sample on every segment boundary --------------------------------------------------------------
    for W, ov in ((128, 0.5), (1000, 0.75)):
        hop = hop_of(W, ov)
        n = 3 * 1000 * hop + 77
        time_bins = int(math.ceil(n / hop))
        step = max(1, int(((time_bins / max(1, time_bins // 1000)) / hop) * hop ** 2))
        x = noise(n, W)
        for k, s in enumerate(range(step, n, step)):
            x[s] = c64([NONFINITE[k % len(NONFINITE)]])[0]
            x[s - 1] = c64([NONFINITE[(k + 1) % len(NONFINITE)]])[0]
        add("segments_W%d_ov%g" % (W, ov), "segments", x, W=W, ov=ov)

    # ---- band-pass: both branches of the preset filters, values at the ends and the tile edges ---------------------------------------
    for bw in (0.1, 0.08):
        m = int(math.ceil(4 / bw)) | 1
        sw = branch_switch(m)
        for n in (sw - 1, sw):
            branch = "fft" if n < sw else "direct"
            where = {"first": 0, "last": n - 1, "head": m // 2, "tail": n - 1 - m // 2, "tile_lo": CONV_TILE - 1, "tile_hi": CONV_TILE}
            for i, (pos, p) in enumerate(where.items()):
                x = noise(n, m + i)
                x[p] = c64([NONFINITE[(i + n) % len(NONFINITE)]])[0]
                add("bandpass_m%d_%s_%s" % (m, branch, pos), "bandpass", x, f_low=0.3, f_high=-0.05, bw=bw)
            add("bandpass_m%d_%s_finite" % (m, branch), "bandpass", noise(n, m), f_low=0.02, f_high=0.12, bw=bw)
            add("bandpass_m%d_%s_huge_1e30" % (m, branch), "bandpass", noise(n, m + 40, 1e30), f_low=0.02, f_high=0.12, bw=bw)
            x = noise(n, m + 41)
            x[n // 3] = c64([(3.4e38, -3.4e38)])[0]
            add("bandpass_m%d_%s_huge_3e38" % (m, branch), "bandpass", x, f_low=0.02, f_high=0.12, bw=bw)
            x = noise(n, m + 42)
            x[[n // 3, n // 2]] = c64([(3.4e38, 0.0), (3.4e38, 0.0)])   # the reference's single-precision FFT overflows
            add("bandpass_m%d_%s_fft_overflow" % (m, branch), "bandpass", x, f_low=0.02, f_high=0.12, bw=bw)
            add("bandpass_m%d_%s_subnormal" % (m, branch), "bandpass", noise(n, m + 43, 1e-42), f_low=0.02, f_high=0.12, bw=bw)
            add("bandpass_m%d_%s_neg_zero" % (m, branch), "bandpass", np.tile(c64([(-0.0, -0.0), (0.0, -0.0)]), n // 2 + 1)[:n],
                f_low=-0.1, f_high=0.1, bw=bw)
    x = noise(5000, 5)
    x[2500] = c64([(INF, 0.0)])[0]
    add("bandpass_m51_fft_n5000_inf", "bandpass", x, f_low=0.02, f_high=0.12, bw=0.08)

    # ---- fft_convolve_1d ---------------------------------------------------------------------------------------------------------------
    rng = np.random.default_rng(77)
    for m in (767, 768, 769):
        h = rng.standard_normal(m) + 1j * rng.standard_normal(m)
        add("convolve_m%d_finite" % m, "convolve", noise(3001, m), h=h)
        x = noise(3001, m + 1)
        x[[0, 1500]] = c64([NONFINITE[m % 6], NONFINITE[(m + 1) % 6]])
        add("convolve_m%d_nonfinite" % m, "convolve", x, h=h)
    hr = rng.standard_normal(51)
    add("convolve_real_real", "convolve", rng.standard_normal(2000), h=hr)
    add("convolve_real_f32", "convolve", rng.standard_normal(2000).astype(np.float32), h=hr.astype(np.float32))
    xr = rng.standard_normal(2000)
    xr[[3, 1999]] = [INF, NAN]
    add("convolve_real_nonfinite", "convolve", xr, h=hr)
    add("convolve_real_x_complex_h", "convolve", rng.standard_normal(2000), h=hr * (1 + 0.5j))
    h = rng.standard_normal(31) + 1j * rng.standard_normal(31)
    h[7] = complex(INF, 0)
    add("convolve_inf_tap", "convolve", noise(2000, 9), h=h)
    h[7] = complex(0, NAN)
    add("convolve_nan_tap", "convolve", noise(2000, 10), h=h)

    # ---- DC correction -----------------------------------------------------------------------------------------------------------------
    for n in (1, 2, 1023, 1024, 1025, EXACT_DC_MAX, EXACT_DC_MAX + 1):
        rng = np.random.default_rng(n)
        base = (rng.standard_normal((n, 2)) + [3.0, -1.5]).astype(np.float32)
        add("dc_n%d_finite" % n, "dc", base)
        x = base.copy()
        x[n // 2, 0] = NAN
        add("dc_n%d_nan_col0" % n, "dc", x)
        x = base.copy()
        x[0, 1], x[n - 1, 1] = INF, -INF
        add("dc_n%d_pm_inf_col1" % n, "dc", x)
        x = base.copy()
        x[:, 0] = np.float32(3e38) * np.where(np.arange(n) % 5 == 4, -0.5, 1.0).astype(np.float32)
        add("dc_n%d_overflow_col0" % n, "dc", x)
        x = base.copy()
        x[:, 0] = np.where(np.arange(n) % 2 == 0, 1e-45, 1e-40).astype(np.float32)
        x[:, 1] = -0.0
        add("dc_n%d_subnormal_negzero" % n, "dc", x)
    for dt in (np.int8, np.uint8, np.int16, np.uint16):
        info = np.iinfo(dt)
        for n in (1, 1025, EXACT_DC_MAX + 1):
            x = np.empty((n, 2), dt)
            x[:, 0] = info.max
            x[:, 1] = np.where(np.arange(n) % 3 == 0, info.min, info.max)
            add("dc_%s_n%d_extremes" % (np.dtype(dt).name, n), "dc", x)

    names = [c.name for c in out]
    assert len(names) == len(set(names)), "case names must be unique"
    return out


GROUPS = ["stft", "segments", "bandpass", "convolve", "dc"]


def segment_bounds(n, W, hop, max_lines=1000):
    """the slices Spectrogram.create_image_segments renders (Spectrogram.py:183-190)"""
    time_bins = int(math.ceil(n / hop))
    step = time_bins / max(1, time_bins // max_lines)
    step = max(1, int((step / hop) * hop ** 2))
    return [(i, min(i + step, n)) for i in range(0, n, step)]


def has_fta(case):
    """export_to_fta is recorded for the small STFT cases (the reference writes it record by record)"""
    return case.group == "stft" and case.W <= 128 and case.ov == 0.5


def answers(case, stft, spectrogram_db, fta, apply_bandpass_filter, fft_convolve_1d, dc_correction):
    """[(kind, array)] of a case through the given functions (the oracle's or the reference's)"""
    if case.group in ("stft", "segments"):
        out = [("stft", stft(case.x, case.W, case.ov)), ("db", spectrogram_db(case.x, case.W, case.ov))]
        if case.group == "segments":
            out += [("db_seg%d" % i, spectrogram_db(case.x[s:e], case.W, case.ov))
                    for i, (s, e) in enumerate(segment_bounds(len(case.x), case.W, hop_of(case.W, case.ov)))]
        if has_fta(case):
            out.append(("fta", fta(case.x, case.W, case.ov)))
        return out
    if case.group == "bandpass":
        return [("out", apply_bandpass_filter(case.x, case.f_low, case.f_high, case.bw))]
    if case.group == "convolve":
        return [("out", fft_convolve_1d(case.x, case.h))]
    return [("out", dc_correction(case.x))]
