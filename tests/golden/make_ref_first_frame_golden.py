"""Regenerates tests/golden/ref_first_frame_{imu,kin}.npz from the REFERENCE ITSELF (oracle/_ref/liblkref.so, the
reference's own eskf.cc / voxel_map.cc / KILO.cc; see make_ref_golden.py). Run where the reference library builds; the
GPU tests (tests/test_gpu_first_frame.py) and the CPU checks (tests/test_first_frame_golden.py) only read the fixtures.

Three KILO::process calls on a fresh node (init_flag_ set), the scene of
test_process_first_frame_then_streaming_frames_match:
  frame 0  the first-frame branch (KILO.cc:331-353) on the raw lidar cloud of first_frame_cases.first_frame_raw_cloud
           (19 k points, regenerated from its seed; stored as raw0_sha256), queue meas0, end0; the reference's x0 / P0 /
           clk0 / acc_norm after StateInitial, the SHA-256 of its world cloud (world0_sha256: the device's must be
           bitwise equal) and its map (map0_digest = mapcmp.digest of the export; the map depends on the cloud alone, so
           both modes store the same digest)
  frames 1-2  streaming frames: the body cloud in the order the reference sorted it (body1, body2), begin / end times,
           the queue, and the reference's x / P / clk, world cloud and n_eff after each frame
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lkref  # noqa: E402
import mapcmp  # noqa: E402
from first_frame_cases import first_frame_raw_cloud, sha256  # noqa: E402
from legkilo_b200 import abi, synth  # noqa: E402


def first_frame(kind):
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=8.0, wall=6.25)
    r = lkref.Reference(cfg, imu_mode_only=(kind == "imu"), gravity=9.81, initialised=False)
    mk = synth.imu_stream if kind == "imu" else synth.kinimu_stream
    raw = first_frame_raw_cloud()
    m0 = mk(49.9, 50.0)
    out = r.process(49.9, 50.0, raw, **{kind: m0})
    assert out["ok"]
    x0, P0, _, c0 = r.get_filter()
    blob0 = r.map_export()
    d = dict(raw0_sha256=sha256(raw), meas0=m0.view(np.uint8), end0=50.0, x0=x0.view(np.float64), P0=P0, clk0=c0.view(np.float64),
             acc_norm=r.acc_norm(), world0_sha256=sha256(out["world"]), map0_digest=mapcmp.digest(blob0))
    t0 = 50.0
    for f in (1, 2):
        rv, tv = synth.random_poses(1, 2e-3, 0.02, stream=8300 + f - 1)
        scan = sc.scan(rotvec=rv[0], trans=tv[0], ext_R=R, ext_t=t, blind=cfg["blind"], stream=8310 + f - 1, n_rings=16, n_az=120,
                       fov_deg=(-15.0, 15.0), streaming=True)
        meas = mk(t0 + 0.001, t0 + 0.13, stream=60 + f - 1)
        out = r.process(t0, t0 + 0.1, scan, **{kind: meas})
        assert out["ok"] and out["n_eff"] > 0.7 * len(scan)
        x, P, _, c = r.get_filter()
        d.update({f"body{f}": out["body"], f"begin{f}": t0, f"meas{f}": meas.view(np.uint8), f"x{f}": x.view(np.float64),
                  f"P{f}": P, f"clk{f}": c.view(np.float64), f"world{f}": out["world"], f"n_eff{f}": out["n_eff"]})
        t0 += 0.1
    np.savez_compressed(os.path.join(HERE, f"ref_first_frame_{kind}.npz"), **d)
    return blob0


if __name__ == "__main__":
    blob_imu = first_frame("imu")
    blob_kin = first_frame("kin")
    assert blob_imu.tobytes() == blob_kin.tobytes()
    print("reference-made first-frame fixtures written")
