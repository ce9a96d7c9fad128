"""Per-phase %globaltimer trace of the fused per-scan kernel at the headline shape (latency diagnosis).

  python tools/trace_fused.py [--workload leg_fusion_b1] [--scans 512] [--launches 48] [--hops] [name=value ...]

Builds bench.py's workload (by default leg_fusion_b1 with its 512-scan ring: inputs larger than L2), warms the ring up
once, then issues --launches back-to-back launches exactly as bench.py does (kernel_timing = 0, so consecutive launches
overlap through programmatic dependent launch). Only those launches carry stamps; each writes its own trace area. The
first of them follows the switch that turns tracing on and is launched without PDL, so it is left out of the figures.
Stamps per block (slots, see lk_fused.cu): 0 entry, 1 first pass starts, per iteration i 14+i pass done,
2+4i block row in shared memory, 3+4i all-reduce total in hand, 4+4i solve done, 20 re-projection stored, 30 loop left,
31 end, 23 / 24 around the first griddepcontrol.wait; a build without the pass-done and re-projection stamps gets the
combined phases printed instead. With finishers (lk_set_param "finishers", on by default) the launch has extra blocks
behind the chunk blocks (workers), which leave at their last row: the finishers' phases of the last exchange (total in
hand, solve, re-projection 20, covariance 21, state stores 22) are printed against the last worker row. Times in
microseconds: medians over the traced launches (min and max beside them) of per-launch medians over blocks, unless the
name says "slowest block" or "last block".

--hops runs the library built with `make -C leg-kilo_b200/csrc HOP_TRACE=1`, whose all-reduce also stamps, per block and
exchange, its chunk row stored (a group leader: level 1 entered), the leader's level-1 sum complete and group row stored, the
total in hand, and its poll rounds per level (lk_llsync.cuh: LL_HOP_SLOTS). Hop 1 runs from the slowest chunk row of a group
to that group's row stored; hop 2 from the last group row stored to the total in hand, for the median and the slowest block.
Poll rounds are the most any lane of the warp took.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("leg-kilo_b200/python", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import legkilo_b200  # noqa: E402
from legkilo_b200 import Engine, _p, abi, lib  # noqa: E402

TRACE_AREA, TRACE_AREAS = 8192, 64  # lk_api.cu
HOP_SLOTS, GROUP, MAX_FINISHERS = 5, 8, 24  # lk_llsync.cuh: LL_HOP_SLOTS, LK_GROUP, LL_MAX_FINISHERS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="leg_fusion_b1")
    ap.add_argument("--scans", type=int, default=0, help="ring size (default: bench.py's)")
    ap.add_argument("--launches", type=int, default=48)
    ap.add_argument("--hops", action="store_true", help="load the hop-trace library (make -C leg-kilo_b200/csrc HOP_TRACE=1) "
                    "and split the all-reduce into its two hops")
    ap.add_argument("param", nargs="*", help="engine parameter name=value (lk_set_param)")
    args = ap.parse_args()
    if args.hops:
        legkilo_b200.LIB_PATH = os.path.join(os.path.dirname(legkilo_b200.LIB_PATH), "liblegkilo_b200_hops.so")
    L = min(args.launches, TRACE_AREAS)
    w = bench.WORKLOADS[args.workload]
    assert w["batch"] == 1, "the fused kernel runs batch-of-one workloads"
    ring = args.scans or w["ring"]
    wl = bench.build_workload(w, 0, ring)
    cfg = wl["cfg"]
    eng = Engine(cfg)
    for kv in args.param:
        k, v = kv.split("=")
        eng.set_param(k, float(v))
    eng.set_param("kernel_timing", 0)
    eng.map_build(wl["map_world"], wl["map_body"])
    eng.stage(wl["x0"], abi.init_cov(ring), abi.process_cov_Q(cfg), np.zeros(ring, abi.CLOCK_DTYPE), wl["pts"], wl["offs"],
              np.zeros(ring))
    for i in range(ring):
        eng.run_range(i, 1, iters=w["iters"])
    eng.sync()
    eng.set_param("trace", 1)
    scans = [(ring // 2 + i) % ring for i in range(L)]
    for s in scans:
        eng.run_range(s, 1, iters=w["iters"])
    eng.sync()
    tr = np.zeros(TRACE_AREA * TRACE_AREAS, np.uint64)
    lib().lk_debug_read(eng.h, 2, _p(tr), tr.nbytes)
    eng.set_param("trace", 0)
    offs = wl["offs"]
    T = []
    NB = []
    H = [] if args.hops else None
    fin_on = dict(kv.split("=") for kv in args.param).get("finishers", "1") != "0"
    import torch
    sms = min(torch.cuda.get_device_properties(0).multi_processor_count, 160)  # lk_fused.cu: fused_max_blocks
    for j, s in enumerate(scans):
        nb = int((offs[s + 1] - offs[s] + 255) // 256)
        grid = nb + (min(sms - nb, MAX_FINISHERS) if fin_on and nb < sms else 0)  # lk_api.cu: fused_args
        NB.append(nb)
        T.append(tr[j * TRACE_AREA: j * TRACE_AREA + grid * 32].reshape(grid, 32).astype(np.int64))
        if args.hops:
            h0 = j * TRACE_AREA + grid * 32 + 64 * 8
            H.append(tr[h0: h0 + nb * 16].reshape(nb, 16).astype(np.int64))
    if args.hops and not any(h.any() for h in H):
        sys.exit("%s wrote no hop stamps: it was built without LK_HOP_TRACE" % legkilo_b200.LIB_PATH)
    it_n = w["iters"]
    us = 1e-3

    def has(b, k):
        return bool((b[:, k] != 0).all())

    rows = {}

    def put(name, v):
        rows.setdefault(name, []).append(v)

    for j in range(1, L):
        nb = NB[j]
        fin = T[j][nb:]  # finishers (none without them)
        b = T[j][:nb]    # workers: the chunk blocks
        t0 = T[j][:, 0].min()
        put("launch: block start spread", (b[:, 0].max() - t0) * us)
        put("prologue (entry -> first pass)", np.median(b[:, 1] - b[:, 0]) * us)
        prev = b[:, 1]
        if has(b, 24):
            put("first griddepcontrol.wait: blocked (median block)", np.median(b[:, 24] - b[:, 23]) * us)
            put("first griddepcontrol.wait: blocked (most)", (b[:, 24] - b[:, 23]).max() * us)
        for it in range(it_n):
            s_row, s_ar, s_sol, s_pass = 2 + 4 * it, 3 + 4 * it, 4 + 4 * it, 14 + it
            if len(fin) and it == it_n - 1:  # the workers leave at their last row; the finishers take it from there
                if has(b, s_pass):
                    put("it%d pass" % it, np.median(b[:, s_pass] - prev) * us)
                put("it%d pass + reduction: slowest worker" % it, (b[:, s_row] - prev).max() * us)
                last_in = b[:, s_row].max()
                put("it%d workers: last row -> last worker end" % it, (b[:, 31].max() - last_in) * us)
                put("finishers: last row -> total in hand (median)", (np.median(fin[:, s_ar]) - last_in) * us)
                put("finishers: solve", np.median(fin[:, s_sol] - fin[:, s_ar]) * us)
                put("finishers: re-projection", np.median(fin[:, 20] - fin[:, s_sol]) * us)
                put("finishers: covariance", np.median(fin[:, 21] - fin[:, 20]) * us)
                put("finishers: state stores (finisher 0)", (fin[0, 22] - fin[0, 21]) * us)
                put("finishers: last row -> last finisher end", (fin[:, 31].max() - last_in) * us)
                put("finishers: start after first worker start (median)", (np.median(fin[:, 0]) - b[:, 0].min()) * us)
                break
            s_row, s_ar, s_sol, s_pass = 2 + 4 * it, 3 + 4 * it, 4 + 4 * it, 14 + it
            if has(b, s_pass):
                put("it%d pass" % it, np.median(b[:, s_pass] - prev) * us)
                put("it%d reduction -> row in smem" % it, np.median(b[:, s_row] - b[:, s_pass]) * us)
            else:
                put("it%d pass + reduction" % it, np.median(b[:, s_row] - prev) * us)
            put("it%d pass: slowest block" % it, (b[:, s_row] - prev).max() * us)
            last_in = b[:, s_row].max()
            put("it%d all-reduce: wait" % it, np.median(b[:, s_ar] - b[:, s_row]) * us)
            put("it%d all-reduce: done after last block row" % it, (np.median(b[:, s_ar]) - last_in) * us)
            put("it%d solve (-> next pass)" % it, np.median(b[:, s_sol] - b[:, s_ar]) * us)
            prev = b[:, s_sol]
            if H is not None:
                h = H[j][:, it * HOP_SLOTS: (it + 1) * HOP_SLOTS]
                lead = np.arange(0, h.shape[0], GROUP)
                last_row = np.array([h[g: g + GROUP, 0].max() for g in lead])  # slowest chunk row of each group (leader: entry)
                put("it%d hop 1: slowest chunk row -> group row stored (median group)" % it, np.median(h[lead, 2] - last_row) * us)
                put("it%d hop 1: slowest chunk row -> group row stored (slowest group)" % it, (h[lead, 2] - last_row).max() * us)
                put("it%d hop 1: of which level-1 sum -> group row stored" % it, np.median(h[lead, 2] - h[lead, 1]) * us)
                put("it%d hop 2: last group row stored -> total in hand (median block)" % it, (np.median(h[:, 3]) - h[lead, 2].max()) * us)
                put("it%d hop 2: last group row stored -> total in hand (slowest block)" % it, (h[:, 3].max() - h[lead, 2].max()) * us)
                put("it%d poll rounds hop 1 (median leader)" % it, np.median(h[lead, 4] & 0xffffffff))
                put("it%d poll rounds hop 1 (most)" % it, (h[lead, 4] & 0xffffffff).max())
                put("it%d poll rounds hop 2 (median block)" % it, np.median(h[:, 4] >> 32))
                put("it%d poll rounds hop 2 (most)" % it, (h[:, 4] >> 32).max())
        if not len(fin):
            if has(b, 20):
                put("re-projection", np.median(b[:, 20] - prev) * us)
                put("after re-projection -> loop left", np.median(b[:, 30] - b[:, 20]) * us)
            else:
                put("re-projection (+ cov)", np.median(b[:, 30] - prev) * us)
            put("block 0 tail (cov update, P store)", (b[0, 31] - b[0, 30]) * us)
        end = T[j][:, 31].max()
        put("launch span (first entry -> last end)", (end - t0) * us)
        if j + 1 < L:
            n = T[j + 1][:NB[j + 1]]
            put("next launch: first block entry - this launch's last end", (n[:, 0].min() - end) * us)
            put("next launch: first exchange done - this launch's last end", (n[:, 3].min() - end) * us)
            put("period (first entry to next first entry)", (T[j + 1][:, 0].min() - t0) * us)
    nbs = sorted({t.shape[0] for t in T})
    print("%s, ring %d, %d traced launches (%d..%d blocks), %s" % (args.workload, ring, L - 1, nbs[0], nbs[-1], bench.gpu_identity(0)))
    for k, v in rows.items():
        v = np.asarray(v)
        print("  %-60s %8.2f  (min %.2f, max %.2f)" % (k, np.median(v), v.min(), v.max()))


if __name__ == "__main__":
    main()
