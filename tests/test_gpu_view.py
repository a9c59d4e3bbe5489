"""GPU suite for the signal view (path_creator.create_path on the device, view.cu): every stream is byte-identical to the numpy
restatement (tests/path_restatement.py, pinned to the reference on the CPU) and the min/max values are bit-identical, on the
pinned cases, on sizes around the kernel's work items (VIEW_ITEM = 4096 samples) and pixel edges, and on a 2^28-sample capture."""
import ctypes as C

import numpy as np
import pytest

import path_restatement as R
import qt_fake

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pc():
    from urh_b200 import _lib

    if not _lib.cuda_available():
        pytest.skip("no CUDA device")
    from urh_b200.cythonext import path_creator

    return path_creator


@pytest.fixture
def ppp():
    from urh_b200 import settings

    old = settings.PIXELS_PER_PATH

    def set_(v):
        settings.PIXELS_PER_PATH = v

    yield set_
    settings.PIXELS_PER_PATH = old


def device_values(x, start, end, spp, stride=1):
    """urh_path_minmax on a device copy of x (stride 2: x becomes column 0 of an (n, 2) array)"""
    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, to_device

    ctx = _lib.default_context()
    host = np.ascontiguousarray(x) if stride == 1 else np.stack([x, np.zeros_like(x)], axis=1)
    d = to_device(host, ctx)
    P = -(-(end - start) // spp)
    out = DeviceArray(ctx, (2 * P,), x.dtype)
    ctx.check(ctx.lib.urh_path_minmax(ctx.handle, C.c_void_p(d.ptr), _lib.dtype_code(x.dtype), stride, len(x), start, end, spp,
                                      C.c_void_p(out.ptr)))
    return out.get()


def bits(a):
    a = np.asarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize])


def column(x):
    from urh_b200.device import DeviceColumn, to_device

    return DeviceColumn(to_device(np.stack([x, np.zeros_like(x)], axis=1)), 0)


def test_streams_and_values_equal_restatement(pc, ppp):
    bad = []
    for cid, x, start, end, ranges, p in R.all_cases():
        ppp(p)
        want, values = R.create_path_streams(x, start, end, ranges, p)
        if pc.create_path_streams(x, start, end, ranges) != want:
            bad.append(cid + " (host)")
        if x.strides[0] != x.itemsize and pc.create_path_streams(column(np.ascontiguousarray(x)), start, end, ranges) != want:
            bad.append(cid + " (DeviceColumn)")
        if values is not None:
            spp = int((end - start) / p)
            if not np.array_equal(bits(device_values(np.ascontiguousarray(x), start, end, spp)), bits(values)):
                bad.append(cid + " (values)")
    assert not bad, bad


def _edge_capture(dtype, n, spp, seed):
    """random samples with NaNs / extremes placed on pixel heads, work-item heads (pixel start + 4096 k) and pixel ends"""
    x = R.random_samples(dtype, n, seed)
    heads = np.arange(0, n, spp)
    items = (heads[:, None] + 4096 * np.arange(1, 4)[None, :]).ravel()
    items = items[items < n]
    ends = heads[1:] - 1
    if np.dtype(dtype).kind == "f":
        b = x.view(np.uint32)
        b[heads[1::7]] = 0x7fc0beef                 # NaN pixel heads
        b[items[::3]] = 0xffc00001                  # NaN heads of later work items: ignored
        x[items[1::3]] = 1e30                       # new maxima exactly on a work-item head
        x[ends[::5]] = -1e30                        # and minima on a pixel's last sample
        x[items[2::3]] = -0.0
    else:
        info = np.iinfo(dtype)
        x[items[::2]] = info.max
        x[ends[::3]] = info.min
        x[heads[2::4]] = info.max
    return x


@pytest.mark.parametrize("spp", [2, 31, 32, 33, 4095, 4096, 4097, 8192, 12289, 50000, 300000])
@pytest.mark.parametrize("dtype", [np.float32, np.int8, np.uint16])
def test_pixels_around_work_items(pc, ppp, spp, dtype):
    p = 64
    ppp(p)
    for r in (0, 1, p - 1):   # the last pixel full, or r samples long
        N = spp * p + r
        x = _edge_capture(dtype, N + 5, spp, spp + r)
        want, values = R.create_path_streams(x, 5, 5 + N, None, p)
        assert int(N / p) == spp
        assert np.array_equal(bits(device_values(x, 5, 5 + N, spp)), bits(values)), (spp, r)
        assert np.array_equal(bits(device_values(x, 5, 5 + N, spp, stride=2)), bits(values)), (spp, r)
        assert pc.create_path_streams(x, 5, 5 + N) == want, (spp, r)


def test_one_pixel_of_the_whole_view(pc, ppp):
    ppp(1)
    x = _edge_capture(np.float32, 3_000_001, 3_000_000, 9)
    want = R.create_path_streams(x, 1, 3_000_001, None, 1)[0]
    assert pc.create_path_streams(x, 1, 3_000_001) == want


def test_device_inputs_equal_host_inputs(pc):
    from urh_b200.device import DeviceColumn, to_device

    iq = R.random_samples(np.int16, 2 * 60_011, 4).reshape(-1, 2)
    d = to_device(iq)
    for col in (0, 1):
        host = pc.create_path_streams(iq[:, col], 11, 60_000, R.epic_ranges(11, 60_000, 9))
        assert pc.create_path_streams(DeviceColumn(d, col), 11, 60_000, R.epic_ranges(11, 60_000, 9)) == host
    q = R.random_samples(np.float32, 70_000, 5)
    for a, b in ((0, 70_000), (3, 9000), (100, 100)):
        assert pc.create_path_streams(to_device(q), a, b) == pc.create_path_streams(q, a, b) == R.create_path_streams(q, a, b)[0]


def test_create_path_under_qt_fake(pc):
    x = R.random_samples(np.float32, 50_000, 6)
    ranges = [(0, 20_000), (60_000, 70_000), (20_000, 50_000)]
    want = R.create_path_streams(x, 0, 50_000, ranges)[0]
    with qt_fake.installed():
        paths = pc.create_path(x, 0, 50_000, ranges)
    assert [p.stream or b"" for p in paths] == want
    assert want[1] == b"" and paths[1].stream is None   # a sub-path past the end is an empty QPainterPath()


def test_plot_data_device_keeps_the_capture_cached(pc):
    from urh_b200.device import DeviceColumn
    from urh_b200.signalprocessing.IQArray import IQArray
    from urh_b200.signalprocessing.Signal import Signal

    sig = Signal("", "view")
    iq = R.random_samples(np.float32, 2 * 40_000, 7).reshape(-1, 2)
    sig.iq_array = IQArray(iq.copy(), _owned=True)
    d1 = sig.iq_array.device()
    re, im = sig.real_plot_data_device, sig.imag_plot_data_device
    assert isinstance(re, DeviceColumn) and len(re) == 40_000 and re.dtype == np.float32
    assert not sig.iq_array._aliased and sig.iq_array.device() is d1
    assert np.array_equal(re.get(), iq[:, 0]) and np.array_equal(im.get(), iq[:, 1])
    assert pc.create_path_streams(im, 0, 40_000) == R.create_path_streams(iq[:, 1], 0, 40_000)[0]


def test_bad_ranges_raise_value_error(pc):
    x = np.zeros(100, np.float32)
    col = column(x)
    for src in (x, col):
        for a, b in ((50, 40), (0, 101), (-1, 10), (101, 101)):
            with pytest.raises(ValueError):
                pc.create_path_streams(src, a, b)
    with pytest.raises(TypeError):
        pc.create_path_streams(np.zeros(100), 0, 100)


def test_capture_of_2_28_samples(pc):
    """a float32 (n, 2) capture of 2^28 samples in HBM, column I, at full view and zoomed views"""
    import torch

    from urh_b200 import _lib
    from urh_b200.device import DeviceArray, DeviceColumn

    n = 1 << 28
    g = torch.Generator(device="cuda").manual_seed(28)
    t = torch.randn((n, 2), device="cuda", dtype=torch.float32, generator=g)
    t[1 << 20, 0] = float("nan")
    t[(1 << 27) + 5, 0] = float("-inf")
    torch.cuda.synchronize()
    ctx = _lib.default_context()
    col = DeviceColumn(DeviceArray(ctx, (n, 2), np.float32, ptr=t.data_ptr(), base=t), 0)
    host = t[:, 0].cpu().numpy()
    for a, b, k in ((0, n, 1), ((1 << 22) + 3, (1 << 22) + 3 + (n >> 6), 40), (n - 9000, n, 3)):
        ranges = R.epic_ranges(a, b, k)
        assert pc.create_path_streams(col, a, b, ranges) == R.create_path_streams(host, a, b, ranges)[0], (a, b)
    del t
