"""Pose-points per second of lk_score_poses against the composition it replaces (the scan staged once per pose with
lk_batch_stage, lk_batch_run(iters=1), n_effective read back with lk_batch_fetch), on the box room (leg_fusion, VLP-16
scans of 16 x 1 800 rays):

  one      one 28 800-point scan x 4 096 poses (a 16 x 16 position grid x 16 yaws around the true pose)
  many     128 scans x 64 poses each (a 4 x 4 position grid x 4 yaws around each scan's pose)

For each: end to end (host clock around the call(s), inputs in host memory, records / counts back in host memory), and
device time (torch.profiler, CUDA kernels only, in a run of their own). Also checks that the counts agree, and prints the
card's name and power limit. Needs a GPU; prints one JSON line at the end.

    python tools/score_poses_timing.py [--reps 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lko  # noqa: E402
import score_cases as sk  # noqa: E402
from legkilo_b200 import Engine, abi, synth  # noqa: E402

CFG = abi.CONFIGS["leg_fusion"]


def workload(kind):
    R, t = abi.extrinsics(CFG)
    sc = synth.BoxScene(ground_half_extent=20.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = lko.Oracle(CFG)
    o.build_voxel_map(pw, pb)
    n_scans, grid, n_yaw = (1, 16, 16) if kind == "one" else (128, 4, 4)
    scans, rot, pos, pset = [], [], [], []
    g = np.linspace(-1.0, 1.0, grid)
    off = np.stack(np.meshgrid(g, g, [0.0], indexing="ij"), -1).reshape(-1, 3)
    for s in range(n_scans):
        rv, tv = (0.0, 0.0, 0.01 * s), (0.05 * s - 3.0, 0.02 * s - 1.0, 0.0)
        scans.append(sc.scan(rotvec=rv, trans=tv, ext_R=R, ext_t=t, blind=CFG["blind"], stream=7000 + s, **synth.VLP16))
        r, p = sk.grid_poses(synth.exp_so3(rv), tv, np.linspace(-0.2, 0.2, n_yaw), off)
        rot.append(r); pos.append(p); pset.append(np.full(len(r), s, np.uint32))
    so = np.concatenate([[0], np.cumsum([len(x) for x in scans])]).astype(np.uint32)
    return o.map_export(), np.concatenate(scans), so, np.concatenate(rot), np.concatenate(pos), np.concatenate(pset)


def score(eng, w):
    _, pts, so, rot, pos, pset = w
    return eng.score_poses(pts, so, pset, rot, pos, sk.ROT_COV, sk.POS_COV)


def composition(eng, w):
    _, pts, so, rot, pos, pset = w
    M = len(rot)
    x = np.concatenate([sk.pose_state(rot[i], pos[i]) for i in range(M)])
    P = np.tile(sk.pose_cov(), (M, 1))
    sizes = (so[1:] - so[:-1]).astype(np.int64)[pset]
    copies = np.concatenate([pts[so[s]:so[s + 1]] for s in pset])
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    eng.stage(x, P, abi.process_cov_Q(CFG), np.zeros(M, abi.CLOCK_DTYPE), copies, offs, np.zeros(M))
    eng.run(iters=1)
    return eng.fetch(want_world=False)["n_eff"]


def host_time(fn, reps):
    fn()  # warm-up: module load, buffer growth
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def kernel_time(fn, out_dir, tag):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
          and "Memset" not in e.name]
    per = {}
    for e in ev:
        per[e.name] = per.get(e.name, 0.0) + e.device_time_total * 1e-3  # us -> ms
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, f"score_{tag}.json"))
    return sum(per.values()), {k[:60]: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:6]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out_dir = os.path.dirname(a.out) if a.out else None
    res = dict(gpu=gpu)
    for kind in ("one", "many"):
        w = workload(kind)
        eng = Engine(CFG)
        eng.map_upload(w[0])
        so, pset = w[2], w[5]
        pp = float(((so[1:] - so[:-1]).astype(np.int64)[pset]).sum())
        rec = score(eng, w)
        n_eff = composition(eng, w)
        agree = bool((rec[:, abi.SCORE_COUNT].astype(np.int64) == n_eff.astype(np.int64)).all())
        e2e_s = host_time(lambda: score(eng, w), a.reps)
        e2e_c = host_time(lambda: composition(eng, w), max(2, a.reps // 2))
        k_s, top_s = kernel_time(lambda: score(eng, w), out_dir, f"{kind}_scorer")
        k_c, top_c = kernel_time(lambda: composition(eng, w), out_dir, f"{kind}_composition")
        assert k_s > 0 and k_c > 0, (top_s, top_c)
        r = dict(poses=len(w[3]), points=int(so[-1]), pose_points=pp, counts_agree=agree,
                 scorer_e2e_s=e2e_s, composition_e2e_s=e2e_c, scorer_kernel_ms=k_s, composition_kernel_ms=k_c,
                 scorer_kernel_rate=pp / (k_s * 1e-3), composition_kernel_rate=pp / (k_c * 1e-3),
                 scorer_e2e_rate=pp / e2e_s[0], composition_e2e_rate=pp / e2e_c[0], scorer_kernels=top_s,
                 composition_kernels=top_c)
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
