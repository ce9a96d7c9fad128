"""Times the front end of the batched path on raw scans: one lk_preprocess_scans call over a whole batch against one
lk_preprocess_scan call per scan of the same batch. Two batches: 128 OS64 scans at leaf 0.5 (the diter shape) and 1 024
VLP-16 scans at leaf 0.3 (leg_fusion), box-room scans in streaming form (curvature = 2 ms time offset).

Each arm is timed around a whole batch with CUDA events on the library's stream (lk_timer_start / lk_timer_stop) and
with the host clock; every call ends in a device synchronise, so both see the whole work. Arms alternate, after
warm-up. --parent-lib times the per-scan arm of another build of the library too (for example the commit before
lk_preprocess_scan went through the batched pipeline), in the same run. Outputs of all arms are compared bit for bit.
Prints the card's name and power limit from the same run, then one JSON line per batch.

    python tools/preprocess_timing.py [--reps R] [--parent-lib PATH] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "leg-kilo_b200", "python"))
import legkilo_b200  # noqa: E402
from legkilo_b200 import abi, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (x.strip() for x in q.split(","))
    return name, limit


class Handle:
    """One handle of the library at `path`, driven through the C ABI with caller-owned, preallocated buffers."""

    def __init__(self, path, cfg):
        L = C.CDLL(path)
        vp, u32 = C.c_void_p, C.c_uint32
        L.lk_create.argtypes = [vp, vp, vp, vp, C.c_int, vp]
        L.lk_destroy.argtypes = [vp]
        L.lk_last_error.restype = C.c_char_p
        L.lk_last_error.argtypes = [vp]
        L.lk_preprocess_scan.argtypes = [vp, vp, u32, C.c_float, vp, vp, vp, vp, vp]
        L.lk_timer_start.argtypes = [vp]
        L.lk_timer_stop.argtypes = [vp] * 5
        if hasattr(L, "lk_preprocess_scans"):
            L.lk_preprocess_scans.argtypes = [vp, u32, vp, vp, C.c_float] + [vp] * 7
        self.L = L
        self._keep = (abi.eskf_cfg(cfg), abi.map_cfg(cfg)) + abi.extrinsics(cfg)
        ec, mc, R, t = self._keep
        self.h = C.c_void_p()
        self._chk(L.lk_create(C.byref(ec), C.byref(mc), _p(R), _p(t), 0, C.byref(self.h)))

    def _chk(self, rc):
        if rc:
            raise RuntimeError(f"error {rc}: {self.L.lk_last_error(self.h).decode()}")

    def timer_start(self):
        self._chk(self.L.lk_timer_start(self.h))

    def timer_stop(self):
        t = C.c_float(); r = C.c_float(); n = C.c_uint32(); nr = C.c_uint32()
        self._chk(self.L.lk_timer_stop(self.h, C.byref(t), C.byref(r), C.byref(n), C.byref(nr)))
        return t.value

    def close(self):
        self.L.lk_destroy(self.h)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Batch:
    def __init__(self, scans, leaf):
        self.scans = scans
        self.leaf = leaf
        self.pts = np.concatenate(scans)
        self.io = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
        self.begin = 100.0 + 0.1 * np.arange(len(scans))
        n, S, w = len(self.pts), len(scans), max(len(s) for s in scans)
        # batch arm outputs
        self.b_pts = np.zeros((n, 4), np.float32); self.so = np.zeros(S + 1, np.uint32); self.sbp = np.zeros(S + 1, np.uint32)
        self.bo = np.zeros(n + 1, np.uint32); self.bc = np.zeros(n, np.float32); self.bt = np.zeros(n)
        # per-scan arm outputs: every scan's results kept, in the batch's layout
        self.s_pts = np.zeros((n, 4), np.float32); self.s_bo = np.zeros(n + S, np.uint32); self.s_bc = np.zeros(n, np.float32)
        self.s_n = np.zeros((S, 2), np.uint32)
        self.w = w

    def run_batch(self, H):
        H._chk(H.L.lk_preprocess_scans(H.h, len(self.scans), _p(self.pts), _p(self.io), self.leaf, _p(self.begin), _p(self.b_pts),
                                       _p(self.so), _p(self.sbp), _p(self.bo), _p(self.bc), _p(self.bt)))

    def run_single(self, H):
        for s, scan in enumerate(self.scans):
            a = int(self.io[s])
            H._chk(H.L.lk_preprocess_scan(H.h, _p(scan), len(scan), self.leaf, _p(self.s_pts[a:]), _p(self.s_n[s, 0:]),
                                          _p(self.s_bo[a + s:]), _p(self.s_bc[a:]), _p(self.s_n[s, 1:])))

    def single_result(self):
        pts, bo, bc = [], [], []
        for s in range(len(self.scans)):
            a, (m, nb) = int(self.io[s]), self.s_n[s]
            pts.append(self.s_pts[a:a + m]); bo.append(self.s_bo[a + s:a + s + nb + 1].copy()); bc.append(self.s_bc[a:a + nb])
        return pts, bo, bc

    def batch_result(self):
        pts, bo, bc = [], [], []
        for s in range(len(self.scans)):
            a, b, ba, bb = int(self.so[s]), int(self.so[s + 1]), int(self.sbp[s]), int(self.sbp[s + 1])
            pts.append(self.b_pts[a:b]); bo.append(self.bo[ba:bb + 1] - a); bc.append(self.bc[ba:bb])
        return pts, bo, bc


def same(r1, r2):
    return all(len(x) == len(y) and all(np.array_equal(a, b) for a, b in zip(x, y)) for x, y in zip(r1, r2))


def raw_scans(n_scans, lidar, distinct=32, stream=9000):
    """n_scans raw scans of the box room at `distinct` different poses, repeated."""
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    rv, tv = synth.random_poses(distinct, 0.2, 2.0, stream=stream)
    base = [sc.scan(rotvec=rv[i], trans=tv[i], ext_R=R, ext_t=t, blind=1.5, stream=stream + 1 + i, streaming=True, **lidar)
            for i in range(distinct)]
    return [base[i % distinct] for i in range(n_scans)]


def measure(batch, arms, reps, warmup=2):
    for _ in range(warmup):
        for _, H, fn in arms:
            fn(H)
    res = {name: dict(device_ms=[], host_ms=[]) for name, _, _ in arms}
    for _ in range(reps):  # arms alternate
        for name, H, fn in arms:
            H.timer_start()
            t = time.perf_counter()
            fn(H)
            host = time.perf_counter() - t
            res[name]["device_ms"].append(H.timer_stop())
            res[name]["host_ms"].append(1e3 * host)
    return {k: dict(device_ms_median=float(np.median(v["device_ms"])), device_ms_min=float(min(v["device_ms"])),
                    host_ms_median=float(np.median(v["host_ms"])), host_ms_min=float(min(v["host_ms"])))
            for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parent-lib", default=None, help="another build of liblegkilo_b200.so: time its per-scan arm too")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    cfg = abi.CONFIGS["leg_fusion"]
    H = Handle(legkilo_b200.LIB_PATH, cfg)
    Hp = Handle(a.parent_lib, cfg) if a.parent_lib else None
    lines = []
    for label, n_scans, lidar, leaf in (("diter_os64_x128", 128, synth.OS64, 0.5), ("leg_fusion_vlp16_x1024", 1024, synth.VLP16, 0.3)):
        B = Batch(raw_scans(n_scans, lidar), leaf)
        arms = [("batch", H, B.run_batch), ("single", H, B.run_single)]
        if Hp:
            arms.append(("single_parent", Hp, B.run_single))
        r = measure(B, arms, a.reps)
        B.run_batch(H); B.run_single(H)
        equal = same(B.batch_result(), B.single_result())
        if Hp:
            B.run_single(Hp)
            equal = equal and same(B.batch_result(), B.single_result())
        out = dict(workload=label, scans=n_scans, points=len(B.pts), leaf=leaf, out_points=int(B.so[-1]),
                   buckets=int(B.sbp[-1]), reps=a.reps, outputs_equal=bool(equal), card=name, power_limit=limit, arms=r)
        for k in r:
            if k != "batch":
                out[f"speedup_vs_{k}"] = r[k]["device_ms_median"] / r["batch"]["device_ms_median"]
        line = json.dumps(out)
        print(line)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    H.close()
    if Hp:
        Hp.close()


if __name__ == "__main__":
    main()
