"""Wall time of one lk_first_frame against the manual first frame it replaces (INTEGRATION.md §3 before the call: StateInitial
and cloudLidarToWorld on the host with numpy, the cloud split into float xyz arrays, then lk_map_build), on raw clouds of a
leg_fusion VLP-16 revolution (16 x 1 800 rays, 28 800 points) and an OS64-shaped one (64 x 2 048 rays, 131 072 points), with
a 0.1 s IMU queue at 400 Hz (39 samples). Both paths end in a device synchronise; each is warmed up on its shapes first, and the two
alternate in the timed repeats. Prints the card's name and power limit, a table, and one JSON line. Needs a GPU.

    python tools/first_frame_timing.py [--repeats 20] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "leg-kilo_b200", "python"))
from legkilo_b200 import Engine, abi, synth  # noqa: E402


def raw_scan(cfg, lidar):
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=40.0, wall=6.25)
    return sc.scan(rotvec=[0.01, -0.02, 0.3], trans=[0.2, -0.1, 0.0], ext_R=R, ext_t=t, blind=0.0, stream=8600, streaming=True,
                   **lidar)


def manual(eng, cfg, x, pts, imu, gravity=9.81):
    """The first frame as a caller wrote it before lk_first_frame."""
    acc, gyr = imu["acc"], imu["gyr"]
    mean_a, mean_w, n = acc[0].copy(), gyr[0].copy(), 1
    for a, w in zip(acc, gyr):
        mean_a += (a - mean_a) / n
        mean_w += (w - mean_w) / n
        n += 1
    acc_norm = np.linalg.norm(mean_a)
    x = x.copy()
    x["grav"][0] = -mean_a / acc_norm * gravity
    x["bw"][0] = mean_w
    x["rot"][0] = np.eye(3).ravel()
    R, t = abi.extrinsics(cfg)
    body = np.ascontiguousarray(pts[:, :3])
    world = ((body.astype(np.float64) @ R.T + t) + x["pos"][0]).astype(np.float32)
    eng.map_build(world, body, R=np.eye(3), rot_cov=1e-6 * np.eye(3), pos_cov=1e-6 * np.eye(3))
    return x, world


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = abi.CONFIGS["leg_fusion"]
    imu = synth.imu_stream(9.9, 10.0)
    x0 = abi.default_states(1)
    res = dict(card=card(), repeats=a.repeats, queue=len(imu), clouds={})
    print(f"card: {res['card']}")
    print(f"{'cloud':>8} {'points':>8} {'lk_first_frame ms':>18} {'manual ms':>10} {'speed-up':>9}")
    for name, lidar in (("vlp16", synth.VLP16), ("os64", synth.OS64)):
        pts = raw_scan(cfg, lidar)
        e_call, e_man = Engine(cfg), Engine(cfg)
        e_call.first_frame(x0, pts, 10.0, imu=imu)  # warm-up: module load, first allocations
        manual(e_man, cfg, x0, pts, imu)
        t_call, t_man = [], []
        for _ in range(a.repeats):
            t = time.perf_counter()
            e_call.first_frame(x0, pts, 10.0, imu=imu)
            t_call.append(time.perf_counter() - t)
            t = time.perf_counter()
            manual(e_man, cfg, x0, pts, imu)
            t_man.append(time.perf_counter() - t)
        mc, mm = float(np.median(t_call)) * 1e3, float(np.median(t_man)) * 1e3
        res["clouds"][name] = dict(points=len(pts), first_frame_ms=mc, manual_ms=mm, speedup=mm / mc,
                                   first_frame_ms_min=min(t_call) * 1e3, manual_ms_min=min(t_man) * 1e3)
        print(f"{name:>8} {len(pts):>8} {mc:>18.3f} {mm:>10.3f} {mm / mc:>8.2f}x")
        e_call.close(); e_man.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
