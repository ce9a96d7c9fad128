"""Writes tests/golden/ref_refine_poses.npz from the reference itself (oracle/_ref/liblkref.so, see make_ref_golden.py): the
exact, near and far poses of tests/golden/ref_score_poses.npz, each refined by K = 5 chained calls of the reference's
KILO::predictUpdatePoint, i.e. the iterated LiDAR update with P held.

The map blob, scan and covariances are read from ref_score_poses.npz. Each call gets a freshly built map (the call inserts
into it; the build is make_ref_score_golden.py's, and its export must equal the stored blob), the state the previous call
left (the pose's state for the first), P = score_cases.pose_cov() reset every time, and both clocks at t (the predict is
then the identity). The pose after every call is stored, with the call's count. The CPU oracle (information-form gain, on
its own import of the stored blob) must follow the same chain: counts equal at every step, poses within 1e-10, which keeps
poses whose points sit at a gate boundary out of the fixture. Writes only this file. Data only.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests", "tests/golden"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lko  # noqa: E402
import lkref  # noqa: E402
import make_ref_score_golden as msg  # noqa: E402
import refine_cases as rk  # noqa: E402
import score_cases as sk  # noqa: E402
from legkilo_b200 import abi  # noqa: E402

CFG = msg.CFG
AGREE = 1e-10


def clock(t):
    clk = np.zeros(1, abi.CLOCK_DTYPE)
    clk["last_predict_time"] = t
    clk["last_update_time"] = t
    return clk


def ref_step(pw, pb, pts, t, x, P):
    r = lkref.Reference(CFG, imu_mode_only=True, gravity=9.81, acc_norm=9.81)
    r.build_voxel_map(pw, pb)
    r.set_filter(x, P, abi.process_cov_Q(CFG), clock(t))
    n = r.predict_update_point(t, pts)["n_eff"]
    return r.get_filter()[0], n


def oracle_step(blob, pts, t, x, P):
    o = lko.Oracle(CFG)
    o.map_import(blob)
    o.set_filter(x, P, abi.process_cov_Q(CFG), clock(t))
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    n = o.predict_update_point(t, pts)["n_eff"]
    return o.get_filter()[0], n


def main():
    d = sk.load_fixture()
    pw, pb, _ = msg.scene()
    r = lkref.Reference(CFG, imu_mode_only=True)
    r.build_voxel_map(pw, pb)
    assert msg.planes_only(r.map_export()).tobytes() == d["blob"].tobytes(), "the scene no longer builds the stored map"
    blob, pts, t = d["blob"], d["pts"], float(d["t"])
    P = sk.pose_cov(d["rot_cov"], d["pos_cov"])
    n = len(rk.POSES)
    rot = np.zeros((n, rk.K + 1, 3, 3)); pos = np.zeros((n, rk.K + 1, 3)); counts = np.zeros((n, rk.K), np.int64)
    for j, i in enumerate(rk.POSES):
        x = sk.pose_state(d["rot"][i], d["pos"][i])
        xo = x.copy()
        rot[j, 0], pos[j, 0] = d["rot"][i], d["pos"][i]
        for k in range(rk.K):
            x, c = ref_step(pw, pb, pts, t, x, P)
            xo, co = oracle_step(blob, pts, t, xo, P)
            assert c == co, (i, k, c, co)
            err = max(np.abs(x["rot"] - xo["rot"]).max(), np.abs(x["pos"] - xo["pos"]).max())
            assert err < AGREE, (i, k, err)
            rot[j, k + 1] = x["rot"][0].reshape(3, 3)
            pos[j, k + 1] = x["pos"][0]
            counts[j, k] = c
    out = os.path.join(HERE, "ref_refine_poses.npz")
    np.savez_compressed(out, poses=rk.POSES, rot=rot, pos=pos, counts=counts)
    print("counts", counts.tolist(), "bytes", os.path.getsize(out))


if __name__ == "__main__":
    main()
