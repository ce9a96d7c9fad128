"""Points per second of lk_map_insert: a box-room trajectory of leg_fusion VLP-16 scans (16 x 1 800 rays, 28 800 points
per scan), one set per scan at the pose it was taken from, inserted on top of the room's first-frame map. Compared with

  cpu      the CPU oracle's map_insert (oracle/lko_insert.py, single thread) on the first --cpu-scans scans;
  buckets  the same points inserted one 2 ms bucket per call (the map-update cost streaming pays per bucket).

Also prints the longest per-root slice of each window (the serial chain of the slice-and-sort insert), the card's name
and its power limit. Needs a GPU; prints one JSON line at the end.

    python tools/map_insert_timing.py [--scans 200] [--cpu-scans 20] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("leg-kilo_b200/python", "oracle"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lko_insert  # noqa: E402
from legkilo_b200 import Engine, abi, synth  # noqa: E402

WINDOW = 32768  # lk_api.cu: MAP_INSERT_WINDOW


def trajectory(cfg, n_scans):
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = lko_insert.Oracle(cfg)
    o.build_voxel_map(pw, pb, np.eye(3), 1e-6 * np.eye(3), 1e-6 * np.eye(3))
    scans, rot, pos = [], [], []
    for i in range(n_scans):
        rv, tv = (0.0, 0.0, 0.002 * i), (0.004 * i, -0.002 * i, 0.0)
        scans.append(sc.scan(rotvec=rv, trans=tv, ext_R=R, ext_t=t, blind=cfg["blind"], stream=3000 + i, streaming=True,
                             **synth.VLP16))
        rot.append(synth.exp_so3(rv)); pos.append(tv)
    so = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    n = len(scans)
    cov = np.tile(1e-6 * np.eye(3), (n, 1, 1))
    return o.map_export(), scans, (np.concatenate(scans), so, np.array(rot), np.array(pos, float), cov, cov)


def longest_slices(cfg, pts, so, rot, pos):
    """Per window, the most points that fall into one root voxel (host restatement of the placement and voxelKeyFloor)."""
    R, t = abi.extrinsics(cfg)
    pi = pts[:, :3].astype(np.float64) @ R.T + t
    set_of = np.repeat(np.arange(len(so) - 1), np.diff(so))
    pw = np.einsum("nij,nj->ni", rot[set_of], pi) + pos[set_of]
    keys = np.floor(pw / float(np.float32(cfg["voxel_size"]))).astype(np.int64)
    out = []
    for a in range(0, len(pts), WINDOW):
        _, cnt = np.unique(keys[a:a + WINDOW], axis=0, return_counts=True)
        out.append(int(cnt.max()))
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--cpu-scans", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cfg = abi.CONFIGS["leg_fusion"]
    blob, scans, args = trajectory(cfg, a.scans)
    pts, so, rot, pos, rc, pc = args
    n = len(pts)
    print(f"trajectory: {a.scans} scans, {n} points ({n / a.scans:.0f} per scan), {(n + WINDOW - 1) // WINDOW} windows")
    # warm-up: module load and first allocations, on a handle of its own
    warm = Engine(cfg)
    warm.map_upload(blob)
    warm.map_insert(pts[:so[2]], so[:3], rot[:2], pos[:2], rc[:2], pc[:2])
    warm.close()

    eng = Engine(cfg)
    eng.map_upload(blob)
    t_call = timed(lambda: eng.map_insert(*args))  # ends in a device synchronise
    st_call = eng.map_stats()

    # one 2 ms bucket per call
    per = []
    for s, scan in enumerate(scans):
        b_pts, b_off, _ = synth.bucketize(scan)
        for b in range(len(b_off) - 1):
            per.append((b_pts[b_off[b]:b_off[b + 1]], s))
    eb = Engine(cfg)
    eb.map_upload(blob)

    def buckets():
        for p, s in per:
            eb.map_insert(p, [0, len(p)], rot[s:s + 1], pos[s:s + 1], rc[s:s + 1], pc[s:s + 1])
    t_buckets = timed(buckets)
    st_buckets = eb.map_stats()

    k = min(a.cpu_scans, a.scans)
    o = lko_insert.Oracle(cfg)
    o.map_import(blob)
    t_cpu = timed(lambda: o.map_insert(pts[:so[k]], so[:k + 1], rot[:k], pos[:k], rc[:k], pc[:k]))

    sl = longest_slices(cfg, pts, so, rot, pos)
    res = dict(card=card(), scans=a.scans, points=n, window=WINDOW, windows=len(sl),
               insert_pts_per_s=n / t_call, insert_s=t_call,
               buckets_pts_per_s=n / t_buckets, buckets_s=t_buckets, bucket_calls=len(per),
               cpu_pts_per_s=int(so[k]) / t_cpu, cpu_scans=k, cpu_s=t_cpu,
               speedup_vs_cpu=(n / t_call) / (int(so[k]) / t_cpu), speedup_vs_buckets=t_buckets / t_call,
               longest_slice_max=max(sl), longest_slice_median=float(np.median(sl)), longest_slices=sl,
               map_call=st_call, map_buckets=st_buckets)
    print(f"card: {res['card']}")
    print(f"lk_map_insert, one call:   {res['insert_pts_per_s'] / 1e6:8.2f} M points/s ({t_call:.3f} s)")
    print(f"one 2 ms bucket per call:  {res['buckets_pts_per_s'] / 1e6:8.2f} M points/s ({t_buckets:.3f} s, {len(per)} calls)")
    print(f"CPU oracle, one thread:    {res['cpu_pts_per_s'] / 1e6:8.2f} M points/s ({k} scans, {t_cpu:.3f} s)")
    print(f"longest per-root slice per window: max {max(sl)}, median {np.median(sl):.0f}")
    print(f"maps: one call {st_call}, per bucket {st_buckets}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
