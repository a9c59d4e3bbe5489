"""GPU (one device): the kernels behind the sharded filters and spectrogram (urh_b200/dist.py), rank by rank on one GPU.
Every shard is run on the window its plan names (its samples plus the halos a neighbour would send), and the concatenated result
must equal the single-GPU public function bit for bit.  The NCCL exchange itself is covered by test_gpu_dist_filter.py."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    from urh_b200 import _lib

    if not _lib.cuda_available():
        pytest.skip("no CUDA device")
    return _lib.default_context()


def complex_capture(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = np.exp(2j * np.pi * 0.05 * t) * (1 + 0.5 * (rng.random(n) > 0.5)) + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64)


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def uneven_bounds(n, world, seed):
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.choice(np.arange(n // (2 * world), n - n // (2 * world)), world - 1, replace=False))
    edges = [0] + [int(c) for c in cuts] + [n]
    return [(edges[i], edges[i + 1]) for i in range(world)]


@pytest.mark.parametrize("m", [1, 10, 101, 1000, 4001, 7])
def test_fir_filter_shard_with_history_equals_whole_capture(ctx, m):
    from urh_b200.cythonext import signal_functions as sf
    from urh_b200.device import DeviceArray, to_device

    rng = np.random.default_rng(m)
    n = 300_001 + 2 * m
    x = complex_capture(n, m)
    taps = ((rng.standard_normal(m) + 1j * rng.standard_normal(m)) / m).astype(np.complex64)
    ref = sf.fir_filter(x, taps)
    d_t = to_device(taps.view(np.float32), ctx)
    for g0 in (max(m - 1, 1), 4096 + 3, 150_000, n - 1025):
        h = m - 1
        d_x = to_device(np.ascontiguousarray(x[g0 - h:]).view(np.float32), ctx)
        out = DeviceArray(ctx, (n - g0,), np.complex64)
        ctx.check(ctx.lib.urh_fir_filter_shard(ctx.handle, C.c_void_p(d_x.ptr + 8 * h), n - g0, 1, C.c_void_p(d_t.ptr), m, C.c_void_p(out.ptr)))
        assert bits_equal(out.get(), ref[g0:]), (m, g0)
    # without history: urh_fir_filter itself
    d_x = to_device(x.view(np.float32), ctx)
    out = DeviceArray(ctx, (n,), np.complex64)
    ctx.check(ctx.lib.urh_fir_filter_shard(ctx.handle, C.c_void_p(d_x.ptr), n, 0, C.c_void_p(d_t.ptr), m, C.c_void_p(out.ptr)))
    assert bits_equal(out.get(), ref)


def test_fir_exact_sass_pinned():
    """the machine code of the instantiation urh_fir_filter launches is pinned: the history mode is a template parameter, so the
    shard entry cannot change it, and any change to the tap loop or the after-loop NaN recheck (k_fir_exact) shows here and has to
    be re-recorded on purpose"""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "fir_exact_sass.json")))
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    lib = os.path.join(ROOT, "urh_b200", "liburh_b200.so")
    if not (os.path.isfile(cuobjdump) and os.path.isfile(nvcc) and os.path.isfile(lib)):
        pytest.skip("cuobjdump / nvcc / the built library not available")
    release = re.search(r"release (\d+\.\d+)", subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout)
    if not release or release.group(1) != golden["nvcc_release"]:
        pytest.skip("the recorded SASS is from nvcc %s" % golden["nvcc_release"])
    sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", sass)
    funcs = {parts[i]: parts[i + 1] for i in range(1, len(parts), 2)}
    body = funcs["_Z11k_fir_exactILb0EEvPK6float2lS2_iPS0_"]
    lines = [ln.strip() for ln in body.splitlines() if re.match(r"/\*[0-9a-f]{4}\*/", ln.strip())]
    import hashlib

    assert len(lines) == golden["instructions"]
    assert hashlib.sha256("\n".join(lines).encode()).hexdigest() == golden["sha256"]


def _dc_sums(ctx, d, n, exact, carry=None):
    s = np.zeros(2, np.float64)
    c = None if carry is None else np.ascontiguousarray(carry, np.float32)
    ctx.check(ctx.lib.urh_dc_column_sums(ctx.handle, C.c_void_p(d.ptr), n, int(exact), c.ctypes.data_as(C.c_void_p) if c is not None else None,
                                         s.ctypes.data_as(C.c_void_p)))
    return s


def _dc_apply(ctx, d, n, mean):
    from urh_b200.device import DeviceArray

    out = DeviceArray(ctx, (n, 2), np.float32)
    ctx.check(ctx.lib.urh_dc_subtract(ctx.handle, C.c_void_p(d.ptr), n, float(mean[0]), float(mean[1]), C.c_void_p(out.ptr)))
    return out.get()


@pytest.mark.parametrize("n", [1, 1000, 3 * 2 ** 20 + 5])
def test_dc_split_exact_order_equals_dc_correction(ctx, n):
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Filter import Filter

    rng = np.random.default_rng(n)
    x = (rng.standard_normal((n, 2)) * 2 + np.array([0.3, -0.7])).astype(np.float32)
    d = to_device(x, ctx)
    whole = _dc_sums(ctx, d, n, True).astype(np.float32)
    # rank-serial hand-over over three pieces continues the same chain
    carry = np.zeros(2, np.float32)
    for a, b in [(0, n // 3), (n // 3, n // 3 + n // 5), (n // 3 + n // 5, n)]:
        carry = _dc_sums(ctx, d[a:b], b - a, True, carry).astype(np.float32)
    assert bits_equal(carry, whole)
    assert bits_equal(whole, np.sum(x, axis=0, dtype=np.float32))
    assert bits_equal(_dc_apply(ctx, d, n, whole / np.float32(n)), Filter.dc_correction(x))


def test_dc_split_double_regime(ctx):
    from urh_b200 import dist as udist
    from urh_b200.device import to_device
    from urh_b200.signalprocessing.Filter import Filter

    n = 5_000_000
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((n, 2)) + np.array([0.123, -0.456])).astype(np.float32)
    d = to_device(x, ctx)
    # one piece: the same reduction as urh_dc_correction
    mean = (_dc_sums(ctx, d, n, False) / n).astype(np.float32)
    assert bits_equal(_dc_apply(ctx, d, n, mean), Filter.dc_correction(x))
    # per-shard double sums folded in rank order: x - float32(float64 mean) (the mean lies far from a float32 rounding midpoint)
    bounds = uneven_bounds(n, 4, 1)
    parts = np.array([_dc_sums(ctx, d[a:b], b - a, False) for a, b in bounds])
    mean = udist.dc_fold_double(parts, n)
    ref_mean = np.mean(x.astype(np.float64), axis=0).astype(np.float32)
    assert bits_equal(mean, ref_mean)
    assert bits_equal(_dc_apply(ctx, d, n, mean), x - ref_mean)


@pytest.mark.parametrize("dtype", [np.int8, np.uint8, np.int16, np.uint16])
def test_dc_split_integer_equals_dc_correction_int(ctx, dtype):
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Filter import Filter

    n = 1_000_003
    info = np.iinfo(dtype)
    x = np.random.default_rng(3).integers(info.min, info.max + 1, (n, 2)).astype(dtype)
    d = to_device(x, ctx)
    total = np.zeros(2, np.int64)
    for a, b in uneven_bounds(n, 3, 2):
        s = np.zeros(2, np.int64)
        ctx.check(ctx.lib.urh_dc_int_column_sums(ctx.handle, C.c_void_p(d[a:b].ptr), _lib.dtype_code(dtype), b - a, s.ctypes.data_as(C.c_void_p)))
        total += s
    assert np.array_equal(total, x.astype(np.int64).sum(axis=0))
    out = DeviceArray(ctx, (n, 2), np.float64)
    ctx.check(ctx.lib.urh_dc_int_subtract(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(dtype), n, float(total[0]) / n, float(total[1]) / n,
                                          C.c_void_p(out.ptr)))
    assert bits_equal(out.get(), Filter.dc_correction(x))


@pytest.mark.parametrize("f_low,f_high,bw", [(0.03, 0.07, 0.08), (0.2, -0.1, 0.42), (-0.7, 0.9, 0.01), (0.1, 0.2, 0.001)])
def test_bandpass_per_rank_windows_equal_single_gpu(ctx, f_low, f_high, bw):
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Filter import Filter

    n = 400_000 if bw >= 0.01 else 120_000
    x = complex_capture(n, 11)
    ref = Filter.apply_bandpass_filter(x, f_low, f_high, bw)
    h = Filter.bandpass_taps(f_low, f_high, bw)
    for world in (2, 4):
        bounds = uneven_bounds(n, world, world)
        plan = udist.bandpass_plan(n, len(h), bounds)
        got = np.concatenate([Filter._convolve_full_slice(x[g0 - left: g1 + right], h, offset, g1 - g0)
                              for (g0, g1), (left, right, offset) in zip(bounds, plan)])
        assert bits_equal(got, ref), (len(h), world)


@pytest.mark.parametrize("W,overlap", [(1024, 0.5), (256, 0.75), (1000, 0.5)])
def test_db_map_per_rank_frames_equal_single_gpu(ctx, W, overlap):
    from urh_b200 import dist as udist
    from urh_b200.device import DeviceArray, to_device
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n = 700_001
    x = complex_capture(n, 21)
    spec = Spectrogram(x, window_size=W, overlap_factor=overlap)
    ref = spec.calculate_spectrogram()
    hop = spec.hop_size
    d_w = to_device(np.hanning(W).astype(np.float64), ctx)
    for world in (2, 3, 4):
        bounds = [(a, b) for a, b in uneven_bounds(n, world, 7 * world)]
        assert any(g0 % hop for g0, _ in bounds[1:])
        plan = udist.frame_plan(n, W, hop, bounds)
        rows = []
        for (g0, g1), (f0, nf, right) in zip(bounds, plan):
            if not nf:
                continue
            win = np.ascontiguousarray(x[f0 * hop: g1 + right])
            d_x = to_device(win.view(np.float32), ctx)
            out = DeviceArray(ctx, (nf, W), np.float32)
            ctx.check(ctx.lib.urh_spectrogram_db(ctx.handle, C.c_void_p(d_x.ptr), len(win), W, hop, C.c_void_p(d_w.ptr), nf, C.c_void_p(out.ptr)))
            rows.append(out.get())
        assert bits_equal(np.concatenate(rows), ref), (W, world)


@pytest.mark.parametrize("W,overlap,transpose", [(1024, 0.5, False), (256, 0.75, True), (1000, 0.5, False)])
def test_image_segments_per_rank_equal_single_gpu(ctx, W, overlap, transpose):
    from urh_b200 import dist as udist
    from urh_b200.signalprocessing.Spectrogram import Spectrogram

    n = 3_000_007
    x = complex_capture(n, 31)
    cmap = np.random.default_rng(4).integers(0, 256, (256, 4)).astype(np.uint8)
    spec = Spectrogram(x, window_size=W, overlap_factor=overlap)
    segments = spec.segment_bounds()
    if transpose:
        ref = [spec.create_spectrogram_image(s, e, transpose=True, colormap=cmap) for s, e, _ in segments]
    else:
        ref = list(spec.create_image_segments(colormap=cmap))
    assert len(ref) >= 4
    bounds = [(0, 1_000_003), (1_000_003, 2_100_001), (2_100_001, n)]   # a segment's tail reaches into the next shard
    segs, owned, rights = udist.segment_plan(n, W, spec.hop_size, bounds)
    assert segs == segments
    got = {}
    for (g0, g1), mine, right in zip(bounds, owned, rights):
        if not mine:
            continue
        local = Spectrogram(x[g0: g1 + right], window_size=W, overlap_factor=overlap)
        for i in mine:
            s, e, _ = segs[i]
            got[i] = local.create_spectrogram_image(s - g0, e - g0, transpose=transpose, colormap=cmap)
    assert sorted(got) == list(range(len(ref)))
    for i, img in enumerate(ref):
        assert bits_equal(got[i], img), i
