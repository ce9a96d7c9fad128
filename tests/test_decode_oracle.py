"""The PointCloud2 decode oracle (lko_decode.decode_pointcloud2: lko.decode_pointcloud2 with the header stamp) pinned to
the reference's own lidar_processing.cc (oracle/lkref_decode.py, skipped without it) and to the fixture made from it (tests/golden/ref_decode.npz): points,
intensity and lidar_begin_time_ / lidar_end_time_ bit for bit, for the three drivers, at filter_num 1 and 3 and blind 0
and 1.5, on the messages of tests/decode_cases.py."""
import os

import numpy as np
import pytest

import decode_cases
import lko_decode
import lkref_decode

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_decode.npz")
NAMES = [m[0] for m in decode_cases.messages()]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_decode_equal(got, ref):
    """(pts, intensity, begin, end) equal bit for bit (NaN points included)."""
    assert got[0].shape == ref[0].shape
    np.testing.assert_array_equal(_bits(got[0]), _bits(ref[0]))
    np.testing.assert_array_equal(_bits(got[1]), _bits(ref[1]))
    np.testing.assert_array_equal(_bits(np.array(got[2:4], np.float64)), _bits(np.array(ref[2:4], np.float64)))


@pytest.mark.skipif(not lkref_decode.available(), reason="needs the reference sources to build oracle/_ref/liblkref_decode.so")
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("combo", range(len(decode_cases.COMBOS)))
def test_oracle_equals_reference(name, combo):
    _, layout, data, ts, stamp = next(m for m in decode_cases.messages() if m[0] == name)
    blind, fn = decode_cases.COMBOS[combo]
    ref = lkref_decode.decode_pointcloud2(data, layout, blind, fn, ts, stamp)
    assert_decode_equal(lko_decode.decode_pointcloud2(data, layout, blind, fn, ts, stamp), ref)
    if name.startswith("box"):
        assert np.isnan(ref[0][:, :3]).any() and len(ref[0]) > 100


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_reference_fixture(name):
    z = np.load(GOLDEN)
    layout = decode_cases.layout_of(z[f"{name}__layout"])
    data, ts, stamp = z[f"{name}__data"], float(z[f"{name}__time_scale"]), float(z[f"{name}__stamp"])
    for c, (blind, fn) in enumerate(decode_cases.COMBOS):
        ref = (z[f"{name}__{c}__pts"], z[f"{name}__{c}__intensity"], *z[f"{name}__{c}__times"])
        assert_decode_equal(lko_decode.decode_pointcloud2(data, layout, blind, fn, ts, stamp), ref)


def test_fixture_covers_ties_and_the_blind_sphere():
    z = np.load(GOLDEN)
    for lt in (1, 2, 3):
        curv = z[f"half{lt}__0__pts"][:, 3] * np.float32(500)
        assert 63 in curv and -63 in curv  # 62.5 and -62.5 rounded away from zero
        # blind 1.5 drops exactly the five points just inside the sphere; the five on it stay
        assert len(z[f"box{lt}__0__pts"]) - len(z[f"box{lt}__2__pts"]) == 5
