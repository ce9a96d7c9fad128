"""Writes tests/golden/ref_score_poses.npz from the reference itself (oracle/_ref/liblkref.so, see make_ref_golden.py): one
scan of the box room scored at 32 poses against a map built by the reference's BuildVoxelMap.

For every pose the reference runs KILO::predictUpdatePoint once, on a freshly built map (the call inserts into it), with
the state at the pose, P = score_cases.pose_cov() and both clocks at t (the predict is then the identity): its
success_pts_size_out is the pose's count. The CPU oracle, fed the reference's exported map, gives the rows at the same
pose; their float64 record (score_cases.row_record) is stored beside the count. The poses:
  exact     the pose the scan was taken from
  near      centimetres / tenths of a degree off
  far       a metre and tens of degrees off
  boundary  pairs of poses 1e-7 m apart along a line across which the reference's count changes (found by bisection): a
            point sits at a gate, radius or voxel boundary between the two
Writes only this file; the other fixtures are untouched. Data only: the map blob (planes, no retained points), the scan,
the poses, counts and sums.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lko  # noqa: E402
import lkref  # noqa: E402
import score_cases as sk  # noqa: E402
from legkilo_b200 import abi, synth  # noqa: E402

CFG = abi.CONFIGS["leg_fusion"]
T = 10.0
SCENE = synth.BoxScene(ground_half_extent=4.0, wall=3.25)
SCAN_POSE = (np.array([0.0, 0.0, 0.0]), np.array([0.0, 0.0, 0.0]))


def scene():
    Re, te = abi.extrinsics(CFG)
    pw, pb = SCENE.map_points(ext_R=Re, ext_t=te, stream=611)
    pts = SCENE.scan(n_rings=8, n_az=110, fov_deg=(-15.0, 15.0), rotvec=SCAN_POSE[0], trans=SCAN_POSE[1], ext_R=Re, ext_t=te,
                     blind=CFG["blind"], stream=612)
    return pw, pb, pts


def ref_count(pw, pb, pts, R, p):
    r = lkref.Reference(CFG, imu_mode_only=True, gravity=9.81, acc_norm=9.81)
    r.build_voxel_map(pw, pb)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = T; clk["last_update_time"] = T
    r.set_filter(sk.pose_state(R, p), sk.pose_cov(), abi.process_cov_Q(CFG), clk)
    return r.predict_update_point(T, pts)["n_eff"]


def oracle_record(blob, pts, R, p):
    o = lko.Oracle(CFG)
    o.map_import(blob)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = T; clk["last_update_time"] = T
    o.set_filter(sk.pose_state(R, p), sk.pose_cov(), abi.process_cov_Q(CFG), clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    r = o.predict_update_point(T, pts, debug=True)
    rec, scale = sk.row_record(r["ok"], r["h"], r["z"], r["R"])
    assert int(rec[abi.SCORE_COUNT]) == r["n_eff"]
    return rec, scale


def planes_only(blob):
    """The map without its retained points (only inserts read them): what a scored pose reads, in a third of the bytes."""
    _, roots, nodes, aux, _ = abi.parse_map_blob(blob)
    aux = aux.copy()
    aux["pts_base"] = 0
    aux["pts_count"] = 0
    aux["pts_cap"] = 0
    return abi.make_map_blob(roots, nodes, aux, np.zeros(0, abi.MAP_POINT_DTYPE))


def boundary_pair(pw, pb, pts, R, p0, direction, length):
    """Two poses 1e-7 m apart on p0 + s * direction, s in [0, length], whose reference counts differ."""
    f = lambda s: ref_count(pw, pb, pts, R, p0 + s * np.asarray(direction))  # noqa: E731
    lo, hi = 0.0, length
    c_lo, c_hi = f(lo), f(hi)
    assert c_lo != c_hi, (c_lo, c_hi)
    while hi - lo > 1e-7:
        mid = 0.5 * (lo + hi)
        c = f(mid)
        if c == c_lo:
            lo = mid
        else:
            hi, c_hi = mid, c
    return [(R, p0 + lo * np.asarray(direction)), (R, p0 + hi * np.asarray(direction))]


def main():
    pw, pb, pts = scene()
    r = lkref.Reference(CFG, imu_mode_only=True)
    r.build_voxel_map(pw, pb)
    blob = planes_only(r.map_export())
    g = synth.rng(613)
    R0, p0 = synth.exp_so3(SCAN_POSE[0]), SCAN_POSE[1]
    poses = [(R0, p0)]
    for _ in range(8):  # near
        poses.append((synth.exp_so3(g.normal(0.0, 0.004, 3)) @ R0, p0 + g.normal(0.0, 0.02, 3)))
    for _ in range(9):  # far
        poses.append((synth.exp_so3(g.uniform(-0.5, 0.5, 3) * np.array([0.3, 0.3, 1.0])) @ R0, p0 + g.uniform(-1.2, 1.2, 3)))
    for _ in range(7):  # boundary pairs
        Rb = synth.exp_so3(g.normal(0.0, 0.003, 3)) @ R0
        d = g.standard_normal(3)
        poses += boundary_pair(pw, pb, pts, Rb, p0 + g.normal(0.0, 0.01, 3), d / np.linalg.norm(d), 0.05)
    assert len(poses) == 32
    rot = np.array([q[0] for q in poses]); pos = np.array([q[1] for q in poses])
    counts = np.array([ref_count(pw, pb, pts, R, p) for R, p in poses], np.int64)
    recs = [oracle_record(blob, pts, R, p) for R, p in poses]
    rec = np.array([a for a, _ in recs]); scale = np.array([b for _, b in recs])
    assert (rec[:, abi.SCORE_COUNT].astype(np.int64) == counts).all(), (rec[:, abi.SCORE_COUNT], counts)
    out = os.path.join(HERE, "ref_score_poses.npz")
    np.savez_compressed(out, blob=blob, pts=pts, rot=rot, pos=pos, rot_cov=sk.ROT_COV, pos_cov=sk.POS_COV, t=T, counts=counts,
                        oracle_record=rec, oracle_scale=scale)
    print("counts", counts.tolist(), "bytes", os.path.getsize(out))


if __name__ == "__main__":
    main()
