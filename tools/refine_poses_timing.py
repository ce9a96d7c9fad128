"""lk_refine_poses against the composition it replaces (the scan staged once per candidate with lk_batch_stage,
lk_batch_run(iters), the refined poses read back with lk_batch_fetch, then lk_score_poses at the refined poses), on the box
room (leg_fusion, VLP-16 scans of 16 x 1 800 rays), 10 iterations:

  one-k     one 28 800-point scan x k candidates (k = 8, 256, 4 096: a position grid x yaws around the true pose)
  many      128 scans x 8 candidates each

For each: end to end (host clock around the call(s), inputs in host memory, poses and records back in host memory), and
device time (torch.profiler, CUDA kernels only, in a run of their own). Also checks that the poses agree, and prints the
card's name and power limit. Needs a GPU; prints one JSON line at the end.

    python tools/refine_poses_timing.py [--reps 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import score_poses_timing as spt  # noqa: E402
import score_cases as sk  # noqa: E402
from legkilo_b200 import Engine, abi, synth  # noqa: E402

CFG = abi.CONFIGS["leg_fusion"]
ITERS = 10


def workload(kind):
    R, t = abi.extrinsics(CFG)
    sc = synth.BoxScene(ground_half_extent=20.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = spt.lko.Oracle(CFG)
    o.build_voxel_map(pw, pb)
    if kind == "many":
        n_scans, grid, n_yaw = 128, 2, 2
    else:
        k = int(kind.split("-")[1])
        n_scans, grid, n_yaw = 1, {8: 2, 256: 8, 4096: 16}[k], {8: 2, 256: 4, 4096: 16}[k]
    scans, rot, pos, pset = [], [], [], []
    g = np.linspace(-0.2, 0.2, grid)
    off = np.stack(np.meshgrid(g, g, [0.0], indexing="ij"), -1).reshape(-1, 3)
    for s in range(n_scans):
        rv, tv = (0.0, 0.0, 0.01 * s), (0.05 * s - 3.0, 0.02 * s - 1.0, 0.0)
        scans.append(sc.scan(rotvec=rv, trans=tv, ext_R=R, ext_t=t, blind=CFG["blind"], stream=7000 + s, **synth.VLP16))
        r, p = sk.grid_poses(synth.exp_so3(rv), tv, np.linspace(-0.03, 0.03, n_yaw), off)
        rot.append(r); pos.append(p); pset.append(np.full(len(r), s, np.uint32))
    so = np.concatenate([[0], np.cumsum([len(x) for x in scans])]).astype(np.uint32)
    return o.map_export(), np.concatenate(scans), so, np.concatenate(rot), np.concatenate(pos), np.concatenate(pset)


def refine(eng, w):
    _, pts, so, rot, pos, pset = w
    return eng.refine_poses(pts, so, pset, rot, pos, sk.ROT_COV, sk.POS_COV, ITERS)


def composition(eng, w):
    _, pts, so, rot, pos, pset = w
    M = len(rot)
    x = np.concatenate([sk.pose_state(rot[i], pos[i]) for i in range(M)])
    P = np.tile(sk.pose_cov(), (M, 1))
    sizes = (so[1:] - so[:-1]).astype(np.int64)[pset]
    copies = np.concatenate([pts[so[s]:so[s + 1]] for s in pset])
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    eng.stage(x, P, abi.process_cov_Q(CFG), np.zeros(M, abi.CLOCK_DTYPE), copies, offs, np.zeros(M))
    eng.run(iters=ITERS)
    xr = eng.fetch(want_world=False)["x"]
    rr = xr["rot"].reshape(M, 3, 3).copy(); pr = xr["pos"].reshape(M, 3).copy()
    return rr, pr, eng.score_poses(pts, so, pset, rr, pr, sk.ROT_COV, sk.POS_COV)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out_dir = os.path.dirname(a.out) if a.out else None
    res = dict(gpu=gpu, iters=ITERS)
    for kind in ("one-8", "one-256", "one-4096", "many"):
        w = workload(kind)
        eng = Engine(CFG)
        eng.map_upload(w[0])
        ro, po, rec = refine(eng, w)
        rc, pc, recc = composition(eng, w)
        pose_diff = float(max(np.abs(ro - rc).max(), np.abs(po - pc).max()))
        counts_agree = bool((rec[:, abi.SCORE_COUNT] == recc[:, abi.SCORE_COUNT]).all())
        e2e_r = spt.host_time(lambda: refine(eng, w), a.reps)
        e2e_c = spt.host_time(lambda: composition(eng, w), max(2, a.reps // 2))
        k_r, top_r = spt.kernel_time(lambda: refine(eng, w), out_dir, f"refine_{kind}")
        k_c, top_c = spt.kernel_time(lambda: composition(eng, w), out_dir, f"refine_{kind}_composition")
        r = dict(poses=len(w[3]), points=int(w[2][-1]), max_pose_diff=pose_diff, counts_agree=counts_agree,
                 refine_e2e_s=e2e_r, composition_e2e_s=e2e_c, e2e_speedup=e2e_c[0] / e2e_r[0], refine_kernel_ms=k_r,
                 composition_kernel_ms=k_c, kernel_ratio=k_c / k_r, refine_kernels=top_r, composition_kernels=top_c)
        print(kind, json.dumps(r), flush=True)
        res[kind] = r
        eng.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
