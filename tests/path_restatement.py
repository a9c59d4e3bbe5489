"""A numpy restatement of path_creator.create_path (path_creator.pyx:19-120), and the cases it is pinned on.

Contract: N = end - start, spp = int(N / PIXELS_PER_PATH).  When spp > 1, pixel k covers [start + k spp, min(start + (k+1) spp, end)),
values[2k], values[2k+1] = its (min, max) as a walk from the pixel's first sample finds them with strict < and > (the first of
equal values wins, NaNs after the first sample are ignored, a NaN first sample is both), x = repeat(arange(start, end, spp), 2)
and scale = float32(N / (2.0 P)).  Otherwise x = arange(start, end), values = samples[start:end], scale = 1.0.  Each sub-path
(a, b) is the Python slice [lo:hi) of x and values with lo = max(0, floor((((a - start) / s) s - 2s) / s)) and
hi = max(0, ceil((((b - start) / s) s + 2s) / s)), in float64 on the float32 scale s.  Its stream is big-endian
{i4 n, n x {i4 1, f8 x, f8 y}, i4 0, i4 0} with y = float64(np.negative(values)), the negation in the sample dtype; an empty
slice has no stream (b"").
"""
import hashlib
import math

import numpy as np

DTYPES = [np.int8, np.uint8, np.int16, np.uint16, np.float32]


def minmax_values(samples, start, end, spp):
    seg = np.asarray(samples[start:end])
    N = len(seg)
    P = -(-N // spp)
    pad = P * spp - N
    fill_lo, fill_hi = (np.inf, -np.inf) if seg.dtype.kind == "f" else (np.iinfo(seg.dtype).max, np.iinfo(seg.dtype).min)
    wide = seg.astype(np.float64) if seg.dtype.kind == "f" else seg.astype(np.int64)
    lo = np.concatenate([np.where(np.isnan(wide), fill_lo, wide) if seg.dtype.kind == "f" else wide, np.full(pad, fill_lo)])
    hi = np.concatenate([np.where(np.isnan(wide), fill_hi, wide) if seg.dtype.kind == "f" else wide, np.full(pad, fill_hi)])
    first = np.arange(P) * spp
    # argmin / argmax return the first occurrence; -0.0 == +0.0 there, as in the walk.  A filled NaN only ties with an
    # infinite extreme, and then the pixel's first sample (index 0, not NaN) already holds it.
    imin = first + np.argmin(lo.reshape(P, spp), axis=1)
    imax = first + np.argmax(hi.reshape(P, spp), axis=1)
    values = np.empty(2 * P, dtype=seg.dtype)
    values[0::2] = seg[imin]
    values[1::2] = seg[imax]
    if seg.dtype.kind == "f":
        head_nan = np.isnan(seg[first])
        values[0::2][head_nan] = seg[first][head_nan]
        values[1::2][head_nan] = seg[first][head_nan]
    return values


def stream(x, y) -> bytes:
    n = len(x)
    if n == 0:
        return b""
    body = np.empty((n, 5), dtype=">u4")
    body[:, 0] = 1
    xb = np.asarray(x, dtype=np.int64).astype(">f8").view(">u4").reshape(n, 2)
    with np.errstate(invalid="ignore"):
        yb = np.negative(np.asarray(y)).astype(">f8").view(">u4").reshape(n, 2)
    body[:, 1:3] = xb
    body[:, 3:5] = yb
    return np.array([n], ">i4").tobytes() + body.tobytes() + np.zeros(2, ">i4").tobytes()


def create_path_streams(samples, start, end, subpath_ranges=None, pixels_per_path=5000):
    """(streams, values or None)"""
    if np.asarray(samples).dtype not in [np.dtype(d) for d in DTYPES]:
        raise TypeError("No matching signature found")
    N = end - start
    spp = int(N / pixels_per_path)
    values = None
    if spp > 1:
        values = minmax_values(samples, start, end, spp)
        x = np.repeat(np.arange(start, end, spp, dtype=np.int64), 2)
        y = values
        s = float(np.float32(N / (2.0 * (len(values) // 2))))
    else:
        x = np.arange(start, end, dtype=np.int64)
        y = np.asarray(samples[start:end])
        s = 1.0
    out = []
    for a, b in ([(start, end)] if subpath_ranges is None else subpath_ranges):
        lo = int(max(0, math.floor(((((a - start) / s) * s) - 2 * s) / s)))
        hi = int(max(0, math.ceil(((((b - start) / s) * s) + 2 * s) / s)))
        out.append(stream(x[lo:hi], y[lo:hi]))
    return out, values


def digest(streams) -> str:
    """sha256 of the exact bytes of every stream and its length (an empty path hashes differently from a missing one)"""
    h = hashlib.sha256()
    for s in streams:
        h.update(len(s).to_bytes(8, "little"))
        h.update(s)
    return h.hexdigest()


# ---- the cases ------------------------------------------------------------------------------------------------------------------
SIZES = [0, 1, 2, 4999, 5000, 9999, 10000, 10001, 14999, 15000, 2 ** 20 + 7]
PAD = 13   # captures are N + PAD long: start 0, 7 (odd) and PAD (the view ends at the capture's end)


def random_samples(dtype, n, seed):
    rng = np.random.default_rng(seed)
    if np.dtype(dtype).kind == "f":
        x = rng.standard_normal(n).astype(np.float32)
        x[rng.integers(0, max(n, 1), n // 50)] = 0.0   # runs of equal values
        return x
    info = np.iinfo(dtype)
    return rng.integers(info.min, int(info.max) + 1, n).astype(dtype)


def capture(dtype, n, layout, seed):
    """1-D samples of n elements: contiguous, or column 0 of an (n, 2) array (element stride 2)"""
    if layout == "contiguous":
        return random_samples(dtype, n, seed)
    iq = random_samples(dtype, 2 * n, seed).reshape(n, 2)
    return iq[:, 0]


def grid_cases():
    """(id, samples, start, end, subpath_ranges, pixels_per_path)"""
    for d in DTYPES:
        for layout in ("contiguous", "stride2"):
            for N in SIZES:
                x = capture(d, N + PAD, layout, N)
                for start in (0, 7, PAD):
                    yield "%s-%s-%d-%d" % (np.dtype(d).name, layout, N, start), x, start, start + N, None, 5000
        for ppp in (1, 7, 65536):
            for N in (0, 1, 2, 6, 13, 4999, 10001, 131073, 2 ** 20 + 7):
                x = capture(d, N + PAD, "contiguous", N + 1)
                yield "%s-ppp%d-%d" % (np.dtype(d).name, ppp, N), x, 7, 7 + N, None, ppp


def special_cases():
    nan_a, nan_b, nan_neg = 0x7fc12345, 0x7f800001, 0xffa00abc   # quiet with payload, signalling, negative signalling
    for spp_n in (10000, 10001, 20000, 100003):   # spp 2, 2, 4, 20
        x = np.random.default_rng(spp_n).standard_normal(spp_n).astype(np.float32)
        spp = int(spp_n / 5000)
        b = x.view(np.uint32)
        # pixel 0: +0 then -0; pixel 1: -0 then +0 (and the rest of both pixels larger in magnitude)
        x[0:spp] = 5.0
        x[0], x[1] = 0.0, -0.0
        x[spp:2 * spp] = 5.0
        x[spp], x[spp + 1] = -0.0, 0.0
        x[2 * spp:3 * spp] = -5.0
        x[2 * spp], x[2 * spp + 1] = -0.0, 0.0
        b[3 * spp] = nan_a                                       # NaN head
        b[4 * spp + spp - 1] = nan_b                             # NaN in the body
        b[5 * spp:6 * spp] = nan_neg                             # a whole pixel of NaN
        b[6 * spp + 1] = 0x7f800000                              # +inf
        b[7 * spp + 1] = 0xff800000                              # -inf
        b[8 * spp:9 * spp] = 0x00000001                          # smallest denormal ...
        b[8 * spp + 1] = 0x807fffff                              # ... and the largest negative denormal
        b[9 * spp] = 0x00400000
        b[10 * spp:11 * spp] = 0x7f800000                        # all +inf after a NaN head
        b[10 * spp] = nan_a
        b[11 * spp:12 * spp] = 0x7f800000                        # +inf head, NaN after it
        b[11 * spp + 1] = nan_b
        b[12 * spp:13 * spp] = 0xff800000                        # -inf pixel with a NaN inside
        b[12 * spp + spp - 1] = nan_neg
        yield "f32-specials-%d" % spp_n, x, 0, spp_n, None, 5000
        yield "f32-specials-raw-%d" % spp_n, x, 0, min(spp_n, 9999), None, 5000   # spp <= 1: every sample straight through
    for d in (np.int8, np.uint8, np.int16, np.uint16):
        info = np.iinfo(d)
        x = np.random.default_rng(3).integers(info.min, int(info.max) + 1, 20011).astype(d)
        x[0:4] = [info.min, info.max, info.min, info.max]
        x[8:12] = info.max
        x[100:110] = info.min
        yield "%s-extremes" % np.dtype(d).name, x, 0, len(x), None, 5000
        yield "%s-extremes-raw" % np.dtype(d).name, x, 3, 9003, None, 5000


def epic_ranges(start, end, n):
    """sub-path ranges shaped like EpicGraphicView._get_sub_path_ranges_and_colors: consecutive tiles of the view"""
    edges = np.linspace(start, end, n + 1).astype(np.int64)
    return [(int(a), int(b)) for a, b in zip(edges[:-1], edges[1:])]


def subpath_cases():
    x = random_samples(np.float32, 1_000_003, 11)
    for N, s0 in ((1_000_000, 3), (9000, 100), (30001, 0)):
        yield "epic-%d" % N, x, s0, s0 + N, epic_ranges(s0, s0 + N, 7), 5000
        yield "outside-%d" % N, x, s0, s0 + N, [(s0 - 50, s0 + 10), (s0 + N - 3, s0 + N + 500), (-1000, -10), (s0 + N + 10, s0 + N + 20),
                                               (s0 + 5, s0 + 5), (s0 + 900, s0 + 100), (s0, s0 + N)], 5000
        yield "many-%d" % N, x, s0, s0 + N, epic_ranges(s0, s0 + N, 2000), 5000
    xi = random_samples(np.int16, 40000, 12)
    yield "epic-int16-stride", np.stack([xi, xi[::-1]], axis=1)[:, 1], 5, 39995, epic_ranges(5, 39995, 13), 5000


def all_cases():
    yield from grid_cases()
    yield from special_cases()
    yield from subpath_cases()
