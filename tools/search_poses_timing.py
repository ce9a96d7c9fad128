"""lk_search_poses against the five-step composition it replaces (the lattice expanded on the host, lk_score_poses with the
wide blocks, the best k per set sorted on the host, lk_refine_poses, lk_score_poses with the tight blocks, the order by
tight count), on the box room (leg_fusion, VLP-16 scans), iters = 10, k = 8:

  recipe-1     1 scan x the recipe grid (31 yaws over +-30 deg x 21 x 21 positions at 0.2 m): 13 671 candidates
  recipe-128   128 scans x the recipe grid: 1.75 M candidates
  fine-16      16 scans x the fine grid (61 yaws at 1 deg x 41 x 41 positions at 0.1 m): 102 541 candidates each

For each: end to end (host clock around the call(s), inputs and outputs in host memory), device time per kernel family
(torch.profiler, CUDA kernels only, in a run of their own), the scorer's scratch after the call (lk_debug_read 4) against
the composition's bytes computed from the header's shapes, and bitwise agreement. Prints the card's name and power limit.
Needs a GPU; prints one JSON line at the end.

    python tools/search_poses_timing.py [--reps 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import score_poses_timing as spt  # noqa: E402
import search_cases as xs  # noqa: E402
from legkilo_b200 import Engine, abi, synth  # noqa: E402

CFG = abi.CONFIGS["leg_fusion"]
ITERS, K = 10, 8
FAMILIES = ("k_score_sum", "k_score", "k_refine_step", "k_search_expand", "k_search_keep", "k_search_gather",
            "k_search_tight", "k_search_rank")


def workload(kind):
    R, t = abi.extrinsics(CFG)
    sc = synth.BoxScene(ground_half_extent=20.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = spt.lko.Oracle(CFG)
    o.build_voxel_map(pw, pb)
    n_scans = {"recipe-1": 1, "recipe-128": 128, "fine-16": 16}[kind]
    if kind.startswith("recipe"):
        att, step, counts = xs.yaw_attitudes(np.arange(-30.0, 30.1, 2.0)), [0.2, 0.2, 1.0], [21, 21, 1]
    else:
        att, step, counts = xs.yaw_attitudes(np.arange(-30.0, 30.1, 1.0)), [0.1, 0.1, 1.0], [41, 41, 1]
    n = (np.asarray(counts) - 1) * np.asarray(step) / 2
    g = synth.rng(7100)
    scans = []
    for s in range(n_scans):
        rv = (0.0, 0.0, np.deg2rad(g.uniform(-20.0, 20.0)))
        tv = (g.uniform(-1.5, 1.5), g.uniform(-1.5, 1.5), 0.0)
        scans.append(sc.scan(rotvec=rv, trans=tv, ext_R=R, ext_t=t, blind=CFG["blind"], stream=7200 + s, **synth.VLP16))
    so = np.concatenate([[0], np.cumsum([len(x) for x in scans])]).astype(np.uint32)
    ao = (np.arange(n_scans + 1) * len(att)).astype(np.uint32)
    origin = np.tile([-n[0], -n[1], 0.0], (n_scans, 1))
    return (o.map_export(), np.ascontiguousarray(np.concatenate(scans), np.float32), so, ao, np.tile(att, (n_scans, 1, 1)),
            origin, np.asarray(step, float), np.asarray(counts, np.uint32))


def search(eng, w):
    _, pts, so, ao, att, origin, step, counts = w
    return eng.search_poses(pts, so, ao, att, origin, step, counts, xs.WIDE_ROT, xs.WIDE_POS, ITERS, xs.TIGHT_ROT,
                            xs.TIGHT_POS, K)


def composition(eng, w):
    _, pts, so, ao, att, origin, step, counts = w
    return xs.compose(eng, pts, so, ao, att, origin, step, counts, ITERS, K)


def composition_bytes(w):
    """Device scratch of the composition's wide lk_score_poses call, from the header's shapes: 16 B per point, 488 B per
    pose, 32 B per (chunk, tile of 16 poses of its set), and the partial rows of one window (at most 64 MiB)."""
    _, pts, so, ao, _, _, _, counts = w
    nc = (so[1:] - so[:-1] + 255) // 256
    cand = (ao[1:] - ao[:-1]).astype(np.int64) * int(np.prod(counts.astype(np.int64)))
    items = int(np.sum(nc.astype(np.int64) * ((cand + 15) // 16)))
    rows = min(int(np.sum(nc.astype(np.int64) * cand)), 1 << 18)
    return 16 * len(pts) + 488 * int(cand.sum()) + 32 * items + 256 * rows


def kernel_split(fn, out_dir, tag):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "Memcpy" in e.name or "Memset" in e.name:
            continue
        fam = next((f for f in FAMILIES if f in e.name), "other")
        per[fam] = per.get(fam, 0.0) + e.device_time_total * 1e-3  # us -> ms
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, f"search_{tag}.json"))
    return sum(per.values()), {k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default="recipe-1,recipe-128,fine-16")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out_dir = os.path.dirname(a.out) if a.out else None
    res = dict(gpu=gpu, iters=ITERS, k=K)
    for kind in a.cases.split(","):
        w = workload(kind)
        eng = Engine(CFG)
        eng.map_upload(w[0])
        out = search(eng, w)
        held = eng.scorer_scratch()
        ref = composition(eng, w)
        e2e_s = spt.host_time(lambda: search(eng, w), a.reps)
        e2e_c = spt.host_time(lambda: composition(eng, w), max(1, a.reps // 2))
        k_s, split_s = kernel_split(lambda: search(eng, w), out_dir, kind)
        k_c, split_c = kernel_split(lambda: composition(eng, w), out_dir, f"{kind}_composition")
        new = sum(v for f, v in split_s.items() if f.startswith("k_search"))
        r = dict(candidates=int(((w[3][1:] - w[3][:-1]).astype(np.int64) * int(np.prod(w[7].astype(np.int64)))).sum()),
                 scans=len(w[2]) - 1, bitwise=xs.same(out, ref), search_e2e_s=e2e_s, composition_e2e_s=e2e_c,
                 e2e_speedup=e2e_c[0] / e2e_s[0], search_kernel_ms=k_s, composition_kernel_ms=k_c,
                 new_kernel_share=new / k_s, search_kernels=split_s, composition_kernels=split_c,
                 search_scratch_bytes=held[0], search_pinned_bytes=held[1],
                 composition_wide_score_bytes=composition_bytes(w))
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
