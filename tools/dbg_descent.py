import sys, os
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("leg-kilo_b200/python","tests","oracle"): sys.path.insert(0, os.path.join(ROOT,p))
import numpy as np, lko, scenes
from legkilo_b200 import Engine, abi, synth
import test_gpu_inputs as T
cfg, blob = T._two_slabs()
g = synth.rng(80); n = 3000
R, t = abi.extrinsics(cfg)
pw = np.c_[g.uniform(-3.8, 3.8, (n, 2)), np.where(np.arange(n) % 2 == 0, 0.12, 0.38) + 0.002 * g.standard_normal(n)]
rot = synth.exp_so3([1e-3, -1e-3, 2e-3]); p = np.array([0.004, -0.003, 0.002])
pts = np.zeros((n, 4), np.float32); pts[:, :3] = synth.world_to_body(pw, rot, p, R, t).astype(np.float32)
x0 = abi.default_states(1); P0 = abi.init_cov(1); Q = abi.process_cov_Q(cfg); clk = np.zeros(1, abi.CLOCK_DTYPE)
for iters in (1, 2, 3):
    ro, xo, Po, _ = T._oracle(cfg, blob, pts, x0, P0, iters)
    res = []
    for params in (dict(fused=1), dict(fused=1), dict(fused=1, slim_p=0), dict(fused=1, lane_cache=0), dict(fused=0)):
        eng = Engine(cfg)
        for k, v in params.items(): eng.set_param(k, v)
        eng.map_upload(blob)
        out = eng.scan_update(x0, P0, Q, clk, pts, [0, len(pts)], [0.0], iters=iters)
        res.append((params, int(out["n_eff"][0]), scenes.state_err(out["x"], xo, Po)))
    print("iters", iters, "oracle", ro["n_eff"], res)
