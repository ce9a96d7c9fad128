"""PointCloud2 messages that pin the decode (lidar_processing.cc:25-108) to the reference: shared by the CPU pin
(tests/test_decode_oracle.py), its fixture (tests/golden/make_ref_decode_golden.py) and the device tests.

Per driver: a slice of a box-room sweep with NaN points and points exactly on (and just inside) the 1.5 m blind sphere;
a short message whose time offsets from the first point are odd multiples of 1/8 s, so that (cur - first) * 500 lands
exactly on .5 (std::round rounds away from zero), on both sides of the first point. For Velodyne also a packed 22-byte
layout (x, y, z, intensity, ring, time at 0/4/8/12/16/18). Every message has a non-zero header stamp."""
import numpy as np

from legkilo_b200 import abi, synth

COMBOS = ((0.0, 1), (0.0, 3), (1.5, 1), (1.5, 3))  # (blind, filter_num)

PACKED22 = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["f4", "f4", "f4", "f4", "u2", "f4"],
                     "offsets": [0, 4, 8, 12, 16, 18], "itemsize": 22})


def layout_array(layout) -> np.ndarray:
    return np.array([layout.point_step, layout.off_x, layout.off_y, layout.off_z, layout.off_intensity, layout.off_time,
                     layout.lidar_type, 0], np.uint32)


def layout_of(arr) -> abi.LkPc2Layout:
    return abi.LkPc2Layout(*[int(v) for v in arr])


def _box(lt):
    msgs, _ = synth.box_pointcloud2s(1, lt, distinct=1, stream=9600 + lt)
    a = msgs[0][8000:9000].copy()
    a["x"][5::97] = np.nan
    a["y"][11::89] = np.nan
    a["z"][17::83] = np.inf
    on = np.array([[1.5, 0, 0], [0, -1.5, 0], [0, 0, 1.5], [1.0, 1.0, 0.5], [-1.0, 0.5, -1.0]], np.float32)
    inside = np.nextafter(on, np.float32(0))
    for k, p in enumerate(np.concatenate([on, inside])):
        i = 40 + 61 * k
        a["x"][i], a["y"][i], a["z"][i] = p
    return a


def _halves(lt):
    """Raw times first + k / 8 s for k in -5..5 (odd k: a tie at .5), in each driver's units and time_scale."""
    k = np.array([0, 1, -1, 3, -3, 5, 2, -5, 7, 4, 1, -1], np.float64)
    n = len(k)
    g = synth.rng(9650 + lt)
    xyz = g.uniform(2.0, 10.0, (n, 3)).astype(np.float32)
    a = np.zeros(n, abi.PC2_DTYPES[lt])
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    a["intensity"] = np.arange(n, dtype=np.float32)
    if lt == 1:
        a["time"] = (0.25 + k / 8).astype(np.float32)  # seconds, time_scale 1
        return a, 1.0
    if lt == 2:
        a["t"] = (64 + k).astype(np.uint32)  # eighths of a second, time_scale 1/8
        return a, 0.125
    a["timestamp"] = 1000.0 + k / 8
    return a, 1.0


def _packed22():
    b = _box(1)[:500]
    a = np.zeros(len(b), PACKED22)
    for f in ("x", "y", "z", "intensity", "ring", "time"):
        a[f] = b[f]
    return a, abi.LkPc2Layout(22, 0, 4, 8, 12, 18, 1, 0)


def messages():
    """[(name, layout, data uint8, time_scale, stamp)]"""
    out = []
    for lt in (1, 2, 3):
        stamp = 1.7e9 + 0.05 * lt
        out.append((f"box{lt}", abi.pc2_layout(lt), _box(lt).view(np.uint8), synth.PC2_TIME_SCALE[lt], stamp))
        a, ts = _halves(lt)
        out.append((f"half{lt}", abi.pc2_layout(lt), a.view(np.uint8), ts, 1.7e9 + 0.0625))
    a, lay = _packed22()
    out.append(("packed22", lay, a.view(np.uint8).reshape(-1), synth.PC2_TIME_SCALE[1], 12.5))
    return out
