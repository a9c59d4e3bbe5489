"""CPU: the .sub export restatement (tests/sub_restatement.py) against the REFERENCE's own IQArray.export_to_sub, byte for byte.

Cases: the five IQ dtypes, alphabets of 2, 3 and 256 values, n = 1..3, entry counts around the 512-entry lines, the 127 / 128 sign
threshold, an armed value that never recurs, float32 NaN / inf / out-of-range samples, int and float frequencies and odd presets, and
a .sub file loaded with Signal and exported again.  The empty and the 1-D capture raise the reference's exception (type and message)
before any file exists, in the product as in the reference.

The reference's answers are recorded in tests/golden/ref_sub_export.json (oracle/cassette.py; regenerate with URH_RECORD_GOLDEN=1
where the reference tree exists)."""
import os

import numpy as np
import pytest

from oracle.cassette import RECORD, Cassette, same
from sub_restatement import body_bound, sub_body, sub_entries, sub_file, u8_column


@pytest.fixture
def cassette(request):
    c = Cassette("sub_export", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ref():
    if not RECORD:
        return None
    from oracle import ref_loader
    return ref_loader.load_python_layer()


def reference_sub(ref, data, path, skip_conversion=False, **kw):
    """the reference's export_to_sub: (file bytes as uint8 or None, (exception type, message, file exists) or None)"""
    if os.path.exists(path):
        os.remove(path)
    try:
        ref.IQArray(data, skip_conversion=skip_conversion).export_to_sub(path, **kw)
    except Exception as e:
        return None, (type(e).__name__, str(e), os.path.exists(path))
    with open(path, "rb") as fh:
        return np.frombuffer(fh.read(), np.uint8), None


def runs_of(values, lengths):
    return np.repeat(np.asarray(values, np.uint8), lengths)


def alternating(entries, a=10, b=200, length=2):
    """`entries` runs of `length` samples alternating between a and b: one entry each"""
    return runs_of([a if i % 2 == 0 else b for i in range(entries)], [length] * entries)


def as_capture(col, dtype, rng):
    """an (n, 2) capture of `dtype` whose convert_to(uint8)[:, 0] is the uint8 column col (Q is noise)"""
    n = len(col)
    col = np.asarray(col, np.uint8)
    if dtype == np.uint8:
        i = col
    elif dtype == np.int8:
        i = (col.astype(np.int16) - 128).astype(np.int8)
    elif dtype == np.uint16:
        i = (col.astype(np.uint16) << 8) | rng.integers(0, 256, n).astype(np.uint16)
    elif dtype == np.int16:
        i = ((col.astype(np.int32) << 8) - 32768 + rng.integers(0, 256, n)).astype(np.int16)
    else:
        i = ((col.astype(np.float32) + 0.5) / 127 - 1).astype(np.float32)
    q = rng.integers(0, 100, n).astype(dtype) if dtype != np.float32 else rng.standard_normal(n).astype(np.float32)
    data = np.stack([i, q], axis=1).astype(dtype)
    assert np.array_equal(u8_column(data), col)
    return data


def seeded_column(n, alphabet, rng, max_run=4):
    vals = rng.choice(256, alphabet, replace=False).astype(np.uint8)
    col = np.repeat(vals[rng.integers(0, alphabet, n)], rng.integers(1, max_run + 1, n))
    return col[:n]


def float_specials():
    x = np.array([np.nan, np.inf, -np.inf, 5.0, -3.0, 1.0, -1.0, 0.0, 1.0 + 1e-7, 2.5e9, -2.5e9, 0.00393, 0.00394] * 7, np.float32)
    x = np.repeat(x, np.arange(len(x)) % 3 + 1)
    return np.stack([x, x[::-1]], axis=1)


def sub_cases():
    rng = np.random.default_rng(2024)
    cases = {}
    for dt in (np.uint8, np.int8, np.uint16, np.int16, np.float32):
        cases["dtype_" + np.dtype(dt).name] = (as_capture(seeded_column(1000, 3, rng), dt, rng), {})
    for k in (2, 3, 256):
        cases["alphabet_%d" % k] = (as_capture(seeded_column(3000, k, rng, max_run=3 if k < 256 else 1), np.uint8, rng), {})
    for n in (1, 2, 3):
        for j, col in enumerate([[7] * n, [200, 7, 200][:n], [7, 7, 200][:n]]):
            cases["n%d_%d" % (n, j)] = (as_capture(col, np.int8, rng), {})
    for e in (511, 512, 513, 1025):
        cases["entries_%d" % e] = (as_capture(alternating(e), np.uint8, rng), {})
    cases["sign_127_128"] = (as_capture(runs_of([127, 128, 127, 128, 126, 129], [3, 2, 1, 5, 2, 1]), np.uint8, rng), {})
    cases["adjacent_200_201"] = (as_capture(runs_of([200, 201, 200, 201], [4, 3, 2, 2]), np.uint8, rng), {})
    cases["never_recurs_first"] = (as_capture(np.r_[[9], alternating(40)].astype(np.uint8), np.uint8, rng), {})
    cases["never_recurs_later"] = (as_capture(np.r_[alternating(6), [9], alternating(9, 11, 12, 3)].astype(np.uint8), np.uint8, rng), {})
    cases["issue_example"] = (as_capture([0, 0, 255, 3, 3], np.uint8, rng), {})
    cases["float_specials"] = (float_specials(), {})
    cases["freq_int"] = (as_capture(seeded_column(100, 2, rng), np.uint8, rng), {"frequency": 868350000})
    cases["freq_float"] = (as_capture(seeded_column(100, 2, rng), np.uint8, rng), {"frequency": 315e6, "preset": "FuriHalSubGhzPreset2FSKDev238Async"})
    cases["odd_preset"] = (as_capture(seeded_column(100, 2, rng), np.uint8, rng), {"frequency": 433.92, "preset": "{x} ünï\tcode  "})
    cases["empty_preset"] = (as_capture(seeded_column(100, 2, rng), np.uint8, rng), {"frequency": -1, "preset": ""})
    return cases


CASES = sub_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference_file(cassette, ref, tmp_path, name):
    data, kw = CASES[name]
    path = str(tmp_path / "ref.sub")
    want, err = cassette.want(lambda: reference_sub(ref, data, path, **kw))
    assert err is None
    mine = np.frombuffer(sub_file(u8_column(data), **kw), np.uint8)
    assert same(mine, want)
    assert len(sub_body(sub_entries(u8_column(data)))) <= body_bound(len(data))


def test_entry_line_breaks():
    for e in (511, 512, 513, 1025):
        body = sub_body(sub_entries(alternating(e)))
        assert body.count(b"\nRAW_Data: ") == (e + 511) // 512
        assert len(body.split()) == e + 2 * ((e + 511) // 512) - (e + 511) // 512


def test_body_bound_is_reached_within_a_small_margin():
    for n in (2, 1000, 4096, 100001):
        col = alternating(n // 2 + 1, 10, 20)[:n]   # "-2" per two samples: the densest body
        used = len(sub_body(sub_entries(col)))
        assert used <= body_bound(n) and body_bound(n) - used <= 48 + 10 + 2


ERROR_CASES = {
    "empty": (np.zeros((0, 2), np.float32), False),
    "empty_int8": (np.zeros((0, 2), np.int8), False),
    "one_dim_float": (np.linspace(-1, 1, 11, dtype=np.float32), True),
    "one_dim_uint8": (np.arange(6, dtype=np.uint8), True),
    "one_dim_empty": (np.zeros(0, np.float32), True),
}


@pytest.mark.parametrize("name", sorted(ERROR_CASES))
def test_errors_match_reference_without_file(cassette, ref, tmp_path, name):
    from urh_b200.signalprocessing.IQArray import IQArray

    data, skip = ERROR_CASES[name]
    path = str(tmp_path / "x.sub")
    want, err = cassette.want(lambda: reference_sub(ref, data, path, skip_conversion=skip))
    assert want is None and err is not None
    with pytest.raises(Exception) as e:
        IQArray(data, skip_conversion=skip).export_to_sub(path)
    assert (type(e.value).__name__, str(e.value), os.path.exists(path)) == tuple(err)


def test_sub_fixture_round_trip(cassette, ref, tmp_path):
    """a .sub file loaded with Signal (Signal.__load_sub_file) and exported again: the reference's file, from the restatement over
    the product's loaded samples"""
    from urh_b200 import settings
    from urh_b200.signalprocessing.Signal import Signal

    path = tmp_path / "remote.sub"
    path.write_text("Filetype: Flipper SubGhz RAW File\nVersion: 1\nFrequency: 433920000\nPreset: FuriHalSubGhzPresetOok650Async\n"
                    "Protocol: RAW\nRAW_Data: 300 -900 300 -300 900 -9000 1 -1 2 -2\nRAW_Data: 450 -450 1350 -100\n")
    out = str(tmp_path / "again.sub")
    settings.write("default_noise_threshold", "3")
    try:
        mine = Signal(str(path), "t")
        data = np.array(mine.iq_array.data)

        def reference():
            sig = ref.Signal(str(path), "t")
            sig.iq_array.export_to_sub(out)
            with open(out, "rb") as fh:
                return np.frombuffer(fh.read(), np.uint8)

        want = cassette.want(reference)
    finally:
        settings.write("default_noise_threshold", "automatic")
    assert same(np.frombuffer(sub_file(u8_column(data)), np.uint8), want)
