"""CPU: the numpy restatement of the device's colormap look-up (bgra_index, tests/bgra_restatement.py) against the reference's
expression, and the inputs of tests/test_gpu_lookup_convert.py shown to separate the look-up's old arithmetic from the reference's:
the range rounded twice (float32 bounds, then their difference) and the 9.0e18 cut-off before the int64 cast.  So the GPU test
can fail, and the current arithmetic is the reference's on every input it uses."""
import numpy as np
import pytest

from bgra_restatement import (ALL_RANGES, DECIMAL_RANGES, F32_BELOW_2_63, REVERSED_RANGES, SPECIAL_VALUES, boundary_values,
                              device_indices, index_values, reference_indices, reference_take, twice_rounded)

ENTRIES = [1, 2, 256, 1024, 1025, 65536, 65537]


def test_decimal_ranges_round_twice():
    """every decimal pair (and its reverse) has a range that float32 bounds round differently; the integer and float32-exact
    pairs do not"""
    for lo, hi in DECIMAL_RANGES + REVERSED_RANGES:
        assert float(np.float32(lo)) != lo and float(np.float32(hi)) != hi, (lo, hi)
        assert twice_rounded(lo, hi), (lo, hi)
    for lo, hi in [(-140, 10), (-80, 10), (-100.5, -20.25)]:
        assert not twice_rounded(lo, hi)


@pytest.mark.parametrize("entries", ENTRIES)
def test_restatement_is_the_reference(entries):
    """the current arithmetic == the reference's expression on every boundary and special value, for every range kind"""
    for lo, hi in ALL_RANGES:
        data = np.concatenate([boundary_values(lo, hi, entries), SPECIAL_VALUES]).reshape(1, -1)
        assert np.array_equal(device_indices(data, entries, lo, hi), reference_indices(data, entries, lo, hi)), (entries, lo, hi)
    idx = index_values(entries).reshape(-1, 3)
    assert np.array_equal(device_indices(idx, entries, normalize=False), reference_indices(idx, entries, normalize=False)), entries


@pytest.mark.parametrize("entries", [256, 1024, 1025, 65536, 65537])
def test_boundary_data_separates_the_double_rounding(entries):
    """on the boundary data of each decimal pair the twice-rounded range picks another entry than the reference somewhere"""
    for lo, hi in DECIMAL_RANGES + REVERSED_RANGES:
        data = boundary_values(lo, hi, entries).reshape(1, -1)
        old = device_indices(data, entries, lo, hi, before_fix=True)
        assert np.any(old != reference_indices(data, entries, lo, hi)), (entries, lo, hi)


def test_cast_cut_off_is_two_to_the_63():
    """numpy casts a float32 exactly below 2^63: 9.0e18, 9.1e18 and the largest float32 below 2^63 take the last entry; 2^63, -2^63,
    NaN and inf take entry 0.  The old 9.0e18 cut-off sent the first three to entry 0."""
    L = 256
    v = np.array([[9.0e18, 9.1e18, F32_BELOW_2_63, 2.0 ** 63, -(2.0 ** 63), np.nan, np.inf, -np.inf]], np.float32)
    want = np.array([L - 1] * 3 + [0] * 5)
    assert np.array_equal(reference_indices(v, L, normalize=False)[:, 0], want)
    assert np.array_equal(device_indices(v, L, normalize=False)[:, 0], want)
    assert np.array_equal(device_indices(v, L, normalize=False, before_fix=True)[:, 0], [0] * 8)
    # normalised values past 9.0e18 reach the cast too: data 1e30 over a range of 1e-3 dB
    d = np.array([[1e13]], np.float32)
    assert reference_indices(d, 2, 0, 1e-6)[0, 0] == 0   # 1e19 >= 2^63 in float32 arithmetic: INT64_MIN
    assert reference_indices(d, 2, 0, 1.1e-6)[0, 0] == 1


def test_reference_take_is_np_take_with_clip():
    """the reference expression on a colormap gives its rows in the order of data.T"""
    cmap = np.arange(40, dtype=np.uint8).reshape(10, 4)
    data = np.array([[0.0, 5.0, 9.0], [-3.0, 100.0, np.nan]], np.float32)
    got = reference_take(data, cmap, 0, 9)
    assert got.shape == (3, 2, 4)
    assert np.array_equal(got[:, :, 0], [[0, 0], [20, 36], [36, 0]])
