"""Times the wire decode of the batched front end: one lk_decode_pointcloud2s call over a whole batch of PointCloud2
messages against one lk_decode_pointcloud2 call per message of the same batch. Two batches: 1 024 VLP-16 messages in the
Velodyne layout (leg_fusion) and 128 OS64 messages in the Ouster layout (diter), box-room sweeps from
synth.box_pointcloud2s, each message in its own pageable host buffer, blind 1.5 m and filter_num 1.

Each arm is timed around a whole batch with CUDA events on the library's stream (lk_timer_start / lk_timer_stop) and
with the host clock; every call ends in a device synchronise, so both see the whole work. Arms alternate, after warm-up.
--parent-lib times the per-message arm of another build of the library too (for example the commit before
lk_decode_pointcloud2 went through the batched pipeline), in the same run. Outputs of all arms are compared bit for bit:
points, intensity, offsets, and begin / end times (the per-message arm's first / last time plus the header stamp).
Prints the card's name and power limit from the same run, then one JSON line per batch.

    python tools/decode_timing.py [--reps R] [--parent-lib PATH] [--out FILE]
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

BLIND, FILTER = 1.5, 1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (x.strip() for x in q.split(","))
    return name, limit


class Handle:
    """One handle of the library at `path`, driven through the C ABI with caller-owned, preallocated buffers."""

    def __init__(self, path, cfg):
        L = C.CDLL(path)
        vp, u32, i32, dbl = C.c_void_p, C.c_uint32, C.c_int32, C.c_double
        L.lk_create.argtypes = [vp, vp, vp, vp, C.c_int, vp]
        L.lk_destroy.argtypes = [vp]
        L.lk_last_error.restype = C.c_char_p
        L.lk_last_error.argtypes = [vp]
        L.lk_decode_pointcloud2.argtypes = [vp, vp, u32, vp, C.c_float, i32, dbl, vp, vp, vp, vp, vp]
        L.lk_timer_start.argtypes = [vp]
        L.lk_timer_stop.argtypes = [vp] * 5
        if hasattr(L, "lk_decode_pointcloud2s"):
            L.lk_decode_pointcloud2s.argtypes = [vp, u32, vp, vp, vp, vp, C.c_float, i32, dbl] + [vp] * 5
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
    def __init__(self, msgs, stamps, lidar_type):
        self.msgs = [m.view(np.uint8) for m in msgs]  # each message its own pageable buffer
        self.stamps = np.ascontiguousarray(stamps, np.float64)
        self.layout = abi.pc2_layout(lidar_type)
        self.ts = synth.PC2_TIME_SCALE[lidar_type]
        self.counts = np.array([len(m) for m in msgs], np.uint32)
        self.ptrs = (C.c_void_p * len(msgs))(*[m.ctypes.data for m in self.msgs])
        self.io = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.uint32)
        n, S = int(self.io[-1]), len(msgs)
        # batch arm outputs
        self.b_pts = np.zeros((n, 4), np.float32); self.b_int = np.zeros(n, np.float32); self.b_off = np.zeros(S + 1, np.uint32)
        self.b_begin = np.zeros(S); self.b_end = np.zeros(S)
        # per-message arm outputs, every message's results kept at its input offset
        self.s_pts = np.zeros((n, 4), np.float32); self.s_int = np.zeros(n, np.float32); self.s_n = np.zeros(S, np.uint32)
        self.s_first = np.zeros(S); self.s_last = np.zeros(S)

    def run_batch(self, H):
        H._chk(H.L.lk_decode_pointcloud2s(H.h, len(self.msgs), self.ptrs, _p(self.counts), _p(self.stamps), C.byref(self.layout),
                                          BLIND, FILTER, self.ts, _p(self.b_pts), _p(self.b_int), _p(self.b_off),
                                          _p(self.b_begin), _p(self.b_end)))

    def run_single(self, H):
        for m, d in enumerate(self.msgs):
            a = int(self.io[m])
            H._chk(H.L.lk_decode_pointcloud2(H.h, _p(d), int(self.counts[m]), C.byref(self.layout), BLIND, FILTER, self.ts,
                                             _p(self.s_pts[a:]), _p(self.s_int[a:]), _p(self.s_n[m:]), _p(self.s_first[m:]),
                                             _p(self.s_last[m:])))

    def batch_result(self):
        return [(self.b_pts[self.b_off[m]:self.b_off[m + 1]], self.b_int[self.b_off[m]:self.b_off[m + 1]], self.b_begin[m],
                 self.b_end[m]) for m in range(len(self.msgs))]

    def single_result(self):
        hesai = self.layout.lidar_type == 3
        return [(self.s_pts[a:a + k], self.s_int[a:a + k], self.s_first[m] if hesai else self.stamps[m] + self.s_first[m],
                 self.s_last[m] if hesai else self.stamps[m] + self.s_last[m])
                for m, (a, k) in enumerate(zip(self.io[:-1].astype(int), self.s_n.astype(int)))]


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view({4: np.uint32, 8: np.uint64}[x.dtype.itemsize])


def same(r1, r2):
    return len(r1) == len(r2) and all(
        len(a[0]) == len(b[0]) and all(np.array_equal(_bits(np.asarray(x)), _bits(np.asarray(y))) for x, y in zip(a, b))
        for a, b in zip(r1, r2))


def measure(arms, reps, warmup=2):
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
    ap.add_argument("--parent-lib", default=None, help="another build of liblegkilo_b200.so: time its per-message arm too")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    cfg = abi.CONFIGS["leg_fusion"]
    H = Handle(legkilo_b200.LIB_PATH, cfg)
    Hp = Handle(a.parent_lib, cfg) if a.parent_lib else None
    lines = []
    for label, n_msgs, lt, lidar in (("velodyne_vlp16_x1024", 1024, 1, synth.VLP16), ("ouster_os64_x128", 128, 2, synth.OS64)):
        msgs, stamps = synth.box_pointcloud2s(n_msgs, lt, lidar=lidar, distinct=32, stream=9800)
        B = Batch(msgs, stamps, lt)
        arms = [("batch", H, B.run_batch), ("single", H, B.run_single)]
        if Hp:
            arms.append(("single_parent", Hp, B.run_single))
        r = measure(arms, a.reps)
        B.run_batch(H); B.run_single(H)
        equal = same(B.batch_result(), B.single_result())
        if Hp:
            B.run_single(Hp)
            equal = equal and same(B.batch_result(), B.single_result())
        out = dict(workload=label, messages=n_msgs, points=int(B.io[-1]), bytes=int(B.io[-1]) * B.layout.point_step,
                   out_points=int(B.b_off[-1]), reps=a.reps, outputs_equal=bool(equal), card=name, power_limit=limit, arms=r)
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
