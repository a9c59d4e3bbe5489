"""The seeded case matrix of the auto-interpretation tests: magnitudes, noise level, segmentation, plateau lengths, median
filter, detect_center, detect_modulation and estimate() at the dtypes, sizes and decision edges where kernels go wrong.

tests/test_autointerp_reference_cpu.py records the reference's answers to every case in tests/golden/ref_autointerp.json and
holds the oracle to them; tests/test_gpu_autointerp.py holds the device to the same answers (``recorded``).  Both build the
cases from here, so the i-th answer of a section belongs to the i-th case."""
import json
import os

import numpy as np

from oracle.cassette import GOLDEN, decode

F32 = np.float32
IQ_DTYPES = (np.int8, np.uint8, np.int16, np.uint16, np.float32)
TILE = 2048   # URH_TILE: the dense pass's tile


def canon(a):
    """float64 copy with every NaN the same NaN (its sign and payload differ between libm and the device)"""
    a = np.asarray(a, dtype=np.float64).copy()
    a[np.isnan(a)] = np.nan
    return a


def recorded(test):
    """the reference's answers recorded by test_autointerp_reference_cpu.<test>, one per case"""
    with open(os.path.join(GOLDEN, "ref_autointerp.json")) as fh:
        return [decode(v) for v in json.load(fh)[test]]


# ---- magnitudes ---------------------------------------------------------------------------------------------------------
def _random_iq(rng, dt, n):
    if dt == np.float32:
        return rng.standard_normal((n, 2)).astype(F32)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, (n, 2), endpoint=True).astype(dt)


EXTREMES = {
    np.int8: [(-128, -128), (127, -128), (0, 0)],
    np.uint8: [(255, 255), (0, 255), (0, 0)],
    np.int16: [(-32768, -32768), (32767, 32767), (-32768, 0)],   # 2 * 2^30 wraps to a negative int32: sqrt -> NaN
    np.uint16: [(65535, 65535), (65535, 0), (0, 0)],
    np.float32: [(np.inf, 0), (np.nan, 1), (-np.inf, np.nan), (1e-45, 1e-45), (1e-40, 0), (1e20, 1e20), (-1e20, 3e19),
                 (3.4e38, 3.4e38), (0, -0.0)],
}


def magnitude_cases():
    rng = np.random.default_rng(101)
    for dt in IQ_DTYPES:
        for n in (0, 1, 2, 3, 255, 256, 257, (1 << 20) + 3):
            iq = _random_iq(rng, dt, n)
            if n >= 3:
                ext = np.array(EXTREMES[dt], dtype=dt)
                iq[:len(ext)] = ext[:n]
                iq[-1] = ext[0]
            yield iq


# ---- noise level ----------------------------------------------------------------------------------------------------------
NOISE_SIZES = (4, 5, 99, 100, 101, 199, 200, 12_345, 1_000_007)


def _chunking(n):
    cs = max(1, int(n * 1 / 100))
    return cs, n // cs


def edge_f32_noise():
    """float32 magnitudes whose second-last 1 % chunk has np.mean == fl(1.1 * min) + 1 ulp: numpy's float32 pairwise sum puts
    it above the quiet edge, a double sum rounded to float32 puts it on the edge (quiet).  The reference returns 0.01."""
    n = 100_000
    rng = np.random.default_rng(150)
    x = (0.011 + 0.0099 * rng.uniform(-1, 1, 1000)).astype(F32)
    x = (x - (x.astype(np.float64).mean() - float(F32(1.1 * F32(0.01))))).astype(F32)
    m = np.ones(n, dtype=F32)
    m[-1000:] = 0.01
    m[-2000:-1000] = x
    return m


def _tie_level():
    """a dyadic minimum chunk mean m whose quiet edge fl32(1.1 * m) has few significant bits, so that a chunk of any size <= 2^10
    filled with that edge value sums exactly in every order"""
    for k in range(1, 4096):
        m = F32(k / 256)
        t = F32(1.1 * m)
        mant, _ = np.frexp(np.float64(t))
        if (mant * 2 ** 12) == np.floor(mant * 2 ** 12):
            return m, t
    raise AssertionError("no short quiet edge")


def noise_cases():
    """(name, magnitudes): float32 and float64 magnitude arrays"""
    rng = np.random.default_rng(202)
    tie_m, tie_t = _tie_level()
    for n in NOISE_SIZES:
        cs, nch = _chunking(n)
        head = n - cs * nch   # samples before the first end-aligned chunk: in no chunk
        loud = 1.0 + 0.05 * rng.random(n)
        quiet = 0.01 + 0.005 * rng.random(n)
        arrays = {}
        a = loud.copy(); a[n - cs:] = quiet[n - cs:]; arrays["quiet_last_chunk"] = a
        a = loud.copy(); a[head:head + cs] = quiet[head:head + cs]; arrays["quiet_first_chunk"] = a
        a = quiet.copy(); a[head:head + cs] = loud[head:head + cs]; arrays["burst_first_chunk"] = a
        a = quiet.copy(); a[n - cs:] = loud[n - cs:]; arrays["burst_last_chunk"] = a
        a = quiet.copy(); a[n // 2:] = loud[n // 2:]; a[:head] = 50.0; arrays["burst_in_head"] = a   # in no chunk: ignored
        arrays["zeros"] = np.zeros(n)
        arrays["constant"] = np.full(n, 0.75)
        a = np.full(n, 9.0); a[n - cs * (nch // 2):] = 10.0; arrays["ratio_0.9_exact"] = a   # min / max == 0.9: not > 0.9
        a = np.full(n, 1.0); a[n - cs:] = tie_m; a[n - 2 * cs:n - cs] = tie_t; arrays["quiet_edge_exact"] = a
        a = np.full(n, 1.0); a[n - cs:] = tie_m
        a[n - 2 * cs:n - cs] = np.nextafter(tie_t, F32(np.inf)); arrays["quiet_edge_above"] = a
        a = loud.copy(); a[n - cs:] = quiet[n - cs:]; a[n // 3] = np.nan; arrays["nan_loud_chunk"] = a
        a = loud.copy(); a[n - cs:] = quiet[n - cs:]; a[n - 1] = np.nan; arrays["nan_quiet_chunk"] = a
        a = loud.copy(); a[n - cs:] = quiet[n - cs:]; a[n // 3] = np.inf; arrays["inf_loud_chunk"] = a
        if head:
            a = loud.copy(); a[n - cs:] = quiet[n - cs:]; a[0] = np.nan; arrays["nan_in_head"] = a
        for name, a in arrays.items():
            for dt in (np.float32, np.float64):
                yield "%s/%d/%s" % (name, n, np.dtype(dt).name), np.ascontiguousarray(a, dtype=dt)
    yield "edge_f32_pairwise", edge_f32_noise()
    yield "edge_f32_pairwise_as_f64", edge_f32_noise().astype(np.float64)


def noise_iq_cases():
    """(name, iq): captures of every IQ dtype with a quiet stretch; the answer is detect_noise_level(get_magnitudes(iq))"""
    rng = np.random.default_rng(303)
    for dt in IQ_DTYPES:
        for n in (5, 101, 199, 12_345, 1_000_007):
            amp = np.where(np.arange(n) < n - max(1, n // 100) * 3, 0.9, 0.02)
            ph = rng.uniform(0, 2 * np.pi, n)
            x = amp * np.exp(1j * ph)
            if dt == np.float32:
                iq = np.stack([x.real, x.imag], 1).astype(F32)
            else:
                info = np.iinfo(dt)
                mid = (int(info.max) + int(info.min) + 1) // 2
                scale = (int(info.max) - mid) * 0.99
                iq = np.clip(np.rint(np.stack([x.real, x.imag], 1) * scale) + mid, info.min, info.max).astype(dt)
            yield "%s/%d" % (np.dtype(dt).name, n), iq


# ---- segmentation ------------------------------------------------------------------------------------------------------
SEG_THR = 0.5


def segment_cases():
    """(name, magnitudes, threshold)"""
    rng = np.random.default_rng(404)
    thr32 = F32(SEG_THR)
    cases = []
    n = 3 * TILE + 7
    for base in (0.0, 1.0):
        other = 1.0 - base
        for L in (9, 10, 11):
            for at in (0, n - L, TILE - L // 2, TILE - L, TILE, 2 * TILE - 1):
                a = np.full(n, base)
                a[at:at + L] = other
                cases.append(("run%d/base%d/at%d" % (L, base, at), a))
    # runs of both classes one after the other, straddling every tile boundary
    a = np.zeros(n)
    pos = 0
    while pos < n:
        L = int(rng.choice([9, 10, 11, 1, 25]))
        a[pos:pos + L] = rng.integers(0, 2)
        pos += L
    cases.append(("mixed_runs", a))
    # exactly the threshold (below), NaN (below), float64 values next to float32(thr)
    a = np.repeat(rng.integers(0, 2, n // 13 + 1).astype(np.float64), 13)[:n]
    a[rng.random(n) < 0.1] = SEG_THR
    cases.append(("equal_thr", a))
    a = np.repeat(rng.integers(0, 2, n // 12 + 1).astype(np.float64), 12)[:n]
    a[rng.random(n) < 0.05] = np.nan
    cases.append(("nan", a))
    up, down = np.nextafter(thr32, F32(2)), np.nextafter(thr32, F32(0))
    between = np.array([float(thr32) + (float(up) - float(thr32)) * f for f in (0.25, 0.5, 0.75)] +
                       [float(thr32) - (float(thr32) - float(down)) * f for f in (0.25, 0.5, 0.75)])
    a = np.repeat(rng.choice(between, n // 11 + 1), 11)[:n]
    cases.append(("f64_between_f32_neighbours", a))
    for m in range(1, 26):
        cases.append(("n%d" % m, np.repeat(rng.integers(0, 2, m), 1).astype(np.float64) * rng.uniform(0.6, 1.4, m)))
    for k in (1, 2, 3):
        for d in (-1, 0, 1):
            m = k * TILE + d
            cases.append(("tiles%d%+d" % (k, d), np.repeat(rng.integers(0, 2, m // 10 + 1), rng.integers(8, 13))[:m].astype(np.float64)))
    # more than 65 536 messages: the wrapper retries with the exact capacity
    a = np.tile(np.r_[np.ones(10), np.zeros(10)], 70_000)
    cases.append(("70000_messages", a))
    for name, a in cases:
        yield name + "/f64", np.ascontiguousarray(a, np.float64), SEG_THR
        if name != "f64_between_f32_neighbours":
            yield name + "/f32", np.ascontiguousarray(a, F32), SEG_THR


# ---- plateau lengths ---------------------------------------------------------------------------------------------------
def plateau_cases():
    """(name, rect float32, center, percentage)"""
    rng = np.random.default_rng(505)
    cases = []
    n = 1003   # pct * n / 100 is no integer for the percentages below (but 0 and 100)
    x = np.repeat(rng.choice([-1.0, 1.0], n // 7 + 1), rng.integers(1, 30, n // 7 + 1))[:n]
    x = np.resize(x, n) + 0.01 * rng.standard_normal(n)
    cases.append(("random", x, 0.0))
    a = x.copy(); a[rng.random(n) < 0.2] = 0.25
    cases.append(("equal_center", a, 0.25))
    a = np.where(np.arange(n) % 17 < 8, -0.0, 1.0)
    cases.append(("minus_zero", a, 0.0))
    a = x.copy(); a[rng.random(n) < 0.05] = np.nan
    cases.append(("nan", a, 0.0))
    cases.append(("single_run", np.full(n, 2.0), 0.0))
    m = 5 * TILE + 3
    cases.append(("across_tiles", np.repeat(np.resize([1.0, -1.0], m // 700 + 1), 700)[:m], 0.0))
    m = 200_001
    cases.append(("200001_plateaus", np.where(np.arange(m) % 2 == 0, 1.0, -1.0), 0.0))   # more than 65 536 plateaus
    for name, a, c in cases:
        for pct in (0, 1, 3, 25, 99, 100):
            yield "%s/%d" % (name, pct), np.ascontiguousarray(a, F32), c, pct


# ---- median filter ------------------------------------------------------------------------------------------------------
MEDIAN_K = (1, 2, 3, 4, 11, 63, 64)


def median_cases():
    """(name, data float64, k); NaN is left out: the order the reference's sort gives NaN is unspecified"""
    rng = np.random.default_rng(606)
    base = {}
    base["random"] = rng.standard_normal(3001)
    f = F32(1.0)
    ulp = float(np.nextafter(f, F32(2))) - 1.0
    base["same_f32"] = 1.0 + rng.choice([-0.3, -0.1, 0.1, 0.3, 0.0], 500) * ulp   # all round to 1.0f (or its neighbours)
    base["signed_zero_inf"] = rng.choice([0.0, -0.0, np.inf, -np.inf, 1.0, -1.0], 400)
    base["short"] = rng.standard_normal(5)
    for name, d in base.items():
        for k in MEDIAN_K:
            yield "%s/%d" % (name, k), np.ascontiguousarray(d), k
    yield "k_gt_n", rng.standard_normal(7), 11


# ---- detect_center -------------------------------------------------------------------------------------------------------
def center_cases():
    """(name, rect float32, max_size)"""
    rng = np.random.default_rng(707)
    for i in range(12):
        n = int(rng.integers(30, 60_000))
        lv = rng.uniform(-2, 2, 2)
        x = (np.repeat(rng.choice(lv, n // 37 + 1), 37)[:n] + rng.standard_normal(n) * rng.uniform(0.005, 0.2)).astype(F32)
        x[rng.random(n) < rng.uniform(0, 0.4)] = -4.0
        yield "random%d" % i, x, (None if i % 3 else 5000)
    yield "constant", np.full(1000, 0.5, F32), None


# ---- modulation ----------------------------------------------------------------------------------------------------------
MOD_PARAMS = {"ASK": [0.3, 1.0], "FSK": [-20e3, 20e3], "PSK": [0.0, np.pi], "OOK": [0.0, 1.0]}


def modulated(oracle, mod, sps, nbits, seed, noise=0.01):
    """complex64 message of `nbits` random bits from the oracle's modulator (pinned to the reference's modulate_c)"""
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 2, nbits).astype(np.uint8)
    bits[0] = 1
    mtype = "ASK" if mod == "OOK" else mod
    iq = oracle.modulate_c(bits, sps, mtype, np.asarray(MOD_PARAMS[mod], F32), 1, 1.0, 10e3, 0.0, 1e6, 0, 0, np.float32)
    x = iq[:, 0].astype(np.float64) + 1j * iq[:, 1]
    x = x + noise * (rng.standard_normal(len(x)) + 1j * rng.standard_normal(len(x)))
    return x.astype(np.complex64)


def modulation_cases(oracle):
    """(name, complex64 message, wavelet_scale, median_filter_order)"""
    seed = 0
    for mod in ("OOK", "ASK", "FSK", "PSK"):
        for sps in (10, 37, 100):
            for k in (10, 12):
                for d in (-1, 0, 1):
                    seed += 1
                    n = (1 << k) + d
                    x = modulated(oracle, mod, sps, n // sps + 2, seed)[:n]
                    scale, order = [(4, 11), (1, 3), (8, 64)][seed % 3]
                    if mod == "OOK":
                        x[np.abs(x) < 0.2] = 0   # the pauses of an on-off keyed message are exact zeros
                    yield "%s/sps%d/n%d/s%d/k%d" % (mod, sps, n, scale, order), x, scale, order
    for scale in (1, 4, 8):
        for n in (4 * scale - 1, 4 * scale, 4 * scale + 1, 8 * scale - 1, 8 * scale, 8 * scale + 1):
            seed += 1
            yield "short/s%d/n%d" % (scale, n), modulated(oracle, "FSK", 3, n, seed)[:n], scale, 11
    for z in range(5):   # 0..4 exact zeros: more than 3 means "OOK" without a transform
        x = modulated(oracle, "FSK", 50, 80, 900 + z)[:4000]
        x[np.arange(z) * 97 + 5] = 0
        yield "zeros%d" % z, x, 4, 11
    for k in (1, 2, 3, 4):   # NaN samples: dropped by |x| > 0, and they count with the zeros
        x = modulated(oracle, "FSK", 50, 80, 910 + k)[:4000]
        x[np.arange(k) * 131 + 7] = complex(np.nan, 0)
        yield "nan%d" % k, x, 4, 11
    x = modulated(oracle, "FSK", 50, 80, 920)[:4000]
    x[[11, 1000]] = [complex(np.nan, 0.0), complex(0.0, np.nan)]
    yield "nan_fsk_2", x, 4, 11
    x = modulated(oracle, "FSK", 50, 80, 921)[:4000]
    x.view(np.float32)[2 * 17:2 * 17 + 2] = [np.inf, np.nan]   # |x| = inf: kept
    yield "inf_nan", x, 4, 11
    for mod in ("ASK", "PSK"):   # lexicographic maximum ties: equal real parts, different imaginary parts
        x = modulated(oracle, mod, 40, 110, 930)[:4096]
        re = np.float32(np.max(x.real))
        x.view(np.float32)[2 * 100:2 * 100 + 2] = [re, -0.5]
        x.view(np.float32)[2 * 2000:2 * 2000 + 2] = [re, 0.7]
        x.view(np.float32)[2 * 3000:2 * 3000 + 2] = [re, 0.2]
        yield "lexmax_tie/%s" % mod, x, 4, 11


def near_threshold(feat, rel=1e-3):
    """recorded features (four variances, fsk, 100-floor peak values, top-ten edge) within `rel` of a decision threshold"""
    if feat is None:
        return False
    v = feat[:4]
    if any(not np.isfinite(x) for x in v):
        return False
    close = lambda a, b: abs(a - b) <= rel * max(abs(a), abs(b), 1e-300)   # noqa: E731
    if any(close(x, 0.15) for x in v):
        return True
    if close(v[0], 1.5 * v[1]) or close(v[0], 10 * v[2]):
        return True
    far_peaks, tenth, eleventh = feat[5], feat[6], feat[7]
    if any(close(p, 100.0) for p in far_peaks):
        return True
    return eleventh is not None and close(tenth, eleventh)


def features_with(cwt_haar, median_filter, data, wavelet_scale, median_filter_order):
    """detect_modulation's quantities built from the given cwt_haar / median_filter (the reference's own while recording):
    (n_nonzero, None) where it returns early, else (n_nonzero, (var_mag, var_norm_mag, var_filtered_mag, var_filtered_norm_mag,
    fsk, far peak values among the ten greatest, 10th greatest, 11th greatest))"""
    n_data = len(data)
    data = data[np.abs(data) > 0]
    if len(data) == 0 or n_data - len(data) > 3:
        return len(data), None
    data = data / np.abs(np.max(data))
    mag = np.abs(cwt_haar(data, scale=wavelet_scale))
    if len(mag) == 0:
        return len(data), None
    norm_mag = np.abs(cwt_haar(data / np.abs(data), scale=wavelet_scale))
    fft = np.abs(np.fft.fftshift(np.fft.fft(data[0: 2 ** int(np.log2(len(data)))])))
    order = np.argsort(fft)[::-1]
    ten = order[0:10]
    far = [float(fft[i]) for i in ten if abs(i - ten[0]) >= 10]
    fsk = any(p >= 100 for p in far)
    return len(data), (float(np.var(mag)), float(np.var(norm_mag)), float(np.var(median_filter(mag, k=median_filter_order))),
                       float(np.var(median_filter(norm_mag, k=median_filter_order))), bool(fsk), far, float(fft[order[min(9, len(order) - 1)]]),
                       float(fft[order[10]]) if len(order) > 10 else None)


# ---- estimate() ---------------------------------------------------------------------------------------------------------
def estimate_cases(oracle):
    """(name, iq): bursts of modulated bits with gaps of noise, every modulation x IQ dtype x bit length x noise level"""
    rng = np.random.default_rng(808)
    i = 0
    for mod in ("OOK", "ASK", "FSK", "PSK"):
        for dt in IQ_DTYPES:
            for sps in (50, 100):
                i += 1
                noise = (0.002, 0.03)[i % 2]
                parts = []
                for burst in range(3):
                    gap = int(rng.integers(2000, 6000))
                    parts.append(noise * (rng.standard_normal(gap) + 1j * rng.standard_normal(gap)))
                    x = modulated(oracle, mod, sps, int(rng.integers(40, 90)), 10_000 + 10 * i + burst, noise)
                    parts.append(x.astype(np.complex128))
                parts.append(noise * (rng.standard_normal(3000) + 1j * rng.standard_normal(3000)))
                x = np.concatenate(parts) * 0.8
                iq = np.stack([x.real, x.imag], 1)
                if dt == np.float32:
                    iq = iq.astype(F32)
                else:
                    info = np.iinfo(dt)
                    mid = (int(info.max) + int(info.min) + 1) // 2
                    iq = np.clip(np.rint(iq * (int(info.max) - mid)) + mid, info.min, info.max).astype(dt)
                yield "%s/%s/sps%d/noise%g" % (mod, np.dtype(dt).name, sps, noise), iq
