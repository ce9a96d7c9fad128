"""Shared by tests/test_first_frame_golden.py (CPU) and tests/test_gpu_first_frame.py: the reference-made first-frame
fixtures, and numpy restatements of the first frame's host steps in the reference's arithmetic (the manual path that
lk_first_frame replaces)."""
import hashlib
import os

import numpy as np

from legkilo_b200 import abi, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def sha256(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def first_frame_raw_cloud():
    """Frame 0's raw lidar cloud (the scene of test_process_first_frame_then_streaming_frames_match): the box room's dense
    first-frame points in the leg_fusion lidar frame, float4 with w = 0. Regenerated from its seed, not stored: the fixtures
    keep its SHA-256 (raw0_sha256) and load_first_frame checks it."""
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    _, pb = synth.BoxScene(ground_half_extent=8.0, wall=6.25).map_points(ext_R=R, ext_t=t)
    return np.concatenate([pb, np.zeros((len(pb), 1), np.float32)], axis=1)


def load_first_frame(kind):
    """tests/golden/ref_first_frame_<kind>.npz (make_ref_first_frame_golden.py) with the structured views restored and
    raw0 regenerated (its hash checked against the one the reference was fed)."""
    d = dict(np.load(os.path.join(GOLD, f"ref_first_frame_{kind}.npz")))
    mdt = abi.IMU_DTYPE if kind == "imu" else abi.KINIMU_DTYPE
    for f in range(3):
        d[f"x{f}"] = d[f"x{f}"].view(abi.STATE_DTYPE)
        d[f"clk{f}"] = d[f"clk{f}"].view(abi.CLOCK_DTYPE)
        d[f"meas{f}"] = d[f"meas{f}"].view(mdt)
    d["raw0"] = first_frame_raw_cloud()
    assert sha256(d["raw0"]) == str(d["raw0_sha256"]), "regenerated frame-0 cloud differs from the one the fixture was made from"
    return d


def first_frame_numpy(meas, gravity):
    """StateInitialByImu / ByKinImu::processing (state_initial.hpp:36-67, :74-105) restated with numpy."""
    acc, gyr = meas["acc"], meas["gyr"]
    mean_a, mean_w, n = acc[0].copy(), gyr[0].copy(), 1
    for a, w in zip(acc, gyr):
        mean_a += (a - mean_a) / n
        mean_w += (w - mean_w) / n
        n += 1
    acc_norm = np.linalg.norm(mean_a)
    return -mean_a / acc_norm * gravity, mean_w, acc_norm


def _mat_vec(M, v, t):
    """M v + t per point in the reference's order, s = 0; s += M_k0 v_0; ... (element-wise numpy: nothing fused)."""
    out = np.empty_like(v)
    for r in range(3):
        s = 0.0 + M[r, 0] * v[:, 0]
        s = s + M[r, 1] * v[:, 1]
        out[:, r] = (s + M[r, 2] * v[:, 2]) + t[r]
    return out


def lidar_to_world_numpy(pts, cfg, pos=(0.0, 0.0, 0.0)):
    """KILO::pointLidarToWorld (KILO.cc:96-106) with rot = I: p_i = R_ext p + t_ext, p_w = I p_i + pos in fp64, rounded to
    float; float4 out with the input's w."""
    R, t = abi.extrinsics(cfg)
    pi = _mat_vec(np.asarray(R, np.float64), pts[:, :3].astype(np.float64), np.asarray(t, np.float64))
    pw = _mat_vec(np.eye(3), pi, np.asarray(pos, np.float64))
    return np.concatenate([pw.astype(np.float32), pts[:, 3:4]], axis=1)


def os64_raw_scan(cfg, stream=8600):
    """One OS64-shaped revolution (64 x 2048 rays, every ray hits the box room, no blind cut): 131 072 raw points, float4
    (x, y, z, time offset)."""
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=40.0, wall=6.25)
    pts = sc.scan(rotvec=[0.01, -0.02, 0.3], trans=[0.2, -0.1, 0.0], ext_R=R, ext_t=t, blind=0.0, stream=stream, streaming=True,
                  **synth.OS64)
    assert len(pts) == 64 * 2048
    return pts


def canonical_map(blob) -> bytes:
    """The map's content as bytes, independent of the storage order the device's atomics gave it: roots by ascending key,
    each octree depth first (children by octant), every node's record and aux with the storage indices (child_base,
    pts_base, parent, pts_cap) and padding zeroed, followed by its retained points. Equal bytes = the same map, bit for bit."""
    _, roots, nodes, aux, pts = abi.parse_map_blob(blob)
    parts = []

    def walk(i):
        n, a = nodes[i:i + 1].copy(), aux[i:i + 1].copy()
        base, cnt = int(a["pts_base"][0]), int(a["pts_count"][0])
        n["child_base"] = 0; n["pad"] = 0
        a["pts_base"] = 0; a["parent"] = 0; a["pts_cap"] = 0; a["pad"] = 0
        parts.extend([n.tobytes(), a.tobytes(), pts[base:base + max(cnt, 0)].tobytes()])
        f = int(nodes[i]["flags"])
        for c in range(8):
            if (f >> abi.NODE_CHILDMASK_SHIFT) & (1 << c):
                walk(int(nodes[i]["child_base"]) + c)

    for r in sorted(roots, key=lambda r: tuple(r["key"])):
        parts.append(r["key"].tobytes())
        walk(int(r["node"]))
    return b"".join(parts)
