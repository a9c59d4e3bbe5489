"""The colormap look-up of the spectrogram images, twice: as the reference evaluates it (Spectrogram.apply_bgra_lookup,
Spectrogram.py:192-206: numpy on a float32 array with Python-scalar bounds), and as the device's bgra_index (spectrogram.cu)
computes it, restated in numpy: float32 subtract, divide, multiply, then the cast to int64 and np.take(mode="clip").

The device restatement can also replay the arithmetic the look-up had before its bounds travelled as doubles: the range formed as
float32(float32(max) - float32(min)) instead of numpy's float32(max - min), and every |v| >= 9.0e18 sent to entry 0 although numpy
casts exactly up to 2^63.  The tests use it to show that their inputs tell the two apart."""
import numpy as np

INT64_MIN = np.iinfo(np.int64).min
F32_BELOW_2_63 = float(np.nextafter(np.float32(2.0 ** 63), np.float32(0)))   # the largest float32 numpy casts to int64 exactly

# (min, max) bounds of each kind: integers (the reference GUI's sliders), float32-exact non-integers, decimals whose range numpy
# rounds once and the old arithmetic twice (searched below), a range of 1e-3, min == max and min > max
INTEGER_RANGES = [(-140, 10), (-80, 10), (-60, -60)]
EXACT_RANGES = [(-100.5, -20.25), (-60.75, 3.5)]
TINY_RANGES = [(-60.3, -60.299)]
EQUAL_RANGES = [(-33.3, -33.3)]


def twice_rounded(lo, hi):
    """whether the range of (lo, hi) rounded once (numpy: float32(hi - lo)) differs from it rounded twice (float32 bounds first)"""
    return np.float32(hi - lo) != np.float32(float(np.float32(hi)) - float(np.float32(lo)))


def twice_rounded_ranges(count, seed=0):
    """`count` (min, max) pairs of one-decimal dB values, min < max, neither a float32, whose two roundings of the range differ"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        lo = int(rng.integers(-1600, -300))
        hi = lo + int(rng.integers(50, 1700))
        if lo % 5 == 0 or hi % 5 == 0:   # d / 10 is a float32 only when d is a multiple of 5
            continue
        pair = (lo / 10, hi / 10)
        if twice_rounded(*pair):
            out.append(pair)
    return out


DECIMAL_RANGES = [(-100.3, -20.7), (-140.1, 10.3)] + twice_rounded_ranges(3, seed=7)
REVERSED_RANGES = [(hi, lo) for lo, hi in DECIMAL_RANGES[:2]]   # min > max
ALL_RANGES = INTEGER_RANGES + EXACT_RANGES + DECIMAL_RANGES + TINY_RANGES + EQUAL_RANGES + REVERSED_RANGES

# data values where float32 arithmetic and the cast go wrong
SPECIAL_VALUES = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, 1e30, -1e30, 3.4028235e38,
                           -3.4028235e38], np.float32)


def index_values(entries):
    """normalize=False data: negative, fractional, at and past the last entry, both sides of the old 9.0e18 cut-off and of 2^63"""
    below_9e18 = float(np.nextafter(np.float32(9.0e18), np.float32(0)))
    return np.array([-1.0, -0.75, -0.0, 0.0, 0.5, 1.0, 1.5, entries - 1.5, entries - 1, entries - 0.5, entries, entries + 0.5, 1e6,
                     2.0 ** 31, 2.0 ** 32, below_9e18, 9.0e18, 9.1e18, F32_BELOW_2_63, 2.0 ** 63, -(2.0 ** 63), -9.1e18, -9.0e18,
                     1e30, np.inf, -np.inf, np.nan], np.float32)


def boundary_values(lo, hi, entries, ulps=2):
    """float32 values on every index boundary lo + k (hi - lo) / (entries - 1), k = 0 .. entries - 1, and up to `ulps` float32
    steps to either side of each"""
    k = np.arange(entries, dtype=np.float64)
    t = (lo + k * ((hi - lo) / max(entries - 1, 1))).astype(np.float32)
    out, up, down = [t], t, t
    for _ in range(ulps):
        up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
        out += [up, down]
    return np.concatenate(out)


def reference_take(data, table, data_min=None, data_max=None, normalize=True):
    """the reference's apply_bgra_lookup, its expression verbatim: np.take(table, ..., mode="clip") of data.T (data float32,
    bounds as given: Python ints or floats)"""
    with np.errstate(all="ignore"):
        if normalize:
            normalized_values = (len(table) - 1) * ((data.T - data_min) / (data_max - data_min))
        else:
            normalized_values = data.T
        return np.take(table, normalized_values.astype(int), axis=0, mode="clip")


def reference_indices(data, entries, data_min=None, data_max=None, normalize=True):
    """the colormap index the reference picks for each pixel of data.T"""
    return reference_take(data, np.arange(entries, dtype=np.int64), data_min, data_max, normalize)


def device_indices(data, entries, data_min=None, data_max=None, normalize=True, before_fix=False):
    """bgra_index of each pixel of data.T: float32 (v - (float)min) / range * (entries - 1), range = (float)(max - min) in double,
    truncated to int64 where |v| < 2^63 and INT64_MIN elsewhere (NaN included), clipped to the table.  before_fix: range =
    (float)((double)(float)max - (double)(float)min) and the 9.0e18 cut-off"""
    v = np.asarray(data, dtype=np.float32).T
    with np.errstate(all="ignore"):
        if normalize:
            if before_fix:
                rng = np.float32(float(np.float32(data_max)) - float(np.float32(data_min)))
            else:
                rng = np.float32(float(data_max) - float(data_min))
            v = np.float32(entries - 1) * ((v - np.float32(data_min)) / rng)
        cut = np.float32(9.0e18) if before_fix else np.float32(2.0 ** 63)
        ok = np.abs(v) < cut
        k = np.where(ok, v, np.float32(0)).astype(np.int64)
    k[~ok] = INT64_MIN
    return np.clip(k, 0, entries - 1)


def distinct_colormap(entries, seed=0):
    """entries x 4 BGRA bytes, the first three bytes distinct for every entry (so that a pixel names its index)"""
    rng = np.random.default_rng(seed)
    idx = np.arange(entries, dtype=np.uint64) * 2654435761 % (1 << 24)
    cmap = np.empty((entries, 4), np.uint8)
    cmap[:, 0], cmap[:, 1], cmap[:, 2] = idx & 255, (idx >> 8) & 255, idx >> 16
    cmap[:, 3] = rng.integers(0, 256, entries)
    return cmap
