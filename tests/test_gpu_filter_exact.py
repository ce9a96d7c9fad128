"""Every filter update the device makes, held against the extended-precision restatement of tests/eskf_exact.py with
bounds scaled to each update's conditioning: lk_update_by_points from explicit rows, a LiDAR bucket through the
batch-of-one kernel, the multi-kernel path and a batch of two (rows from lk_debug_residuals at the same prior, the bucket
stamped at the clock so that its predict is the identity), lk_obs_imu / lk_obs_kinimu with one sample at the clock, and
lk_predict in its four modes. The counts are compared exactly; every ratio is printed (pytest -s)."""
import functools

import numpy as np
import pytest

import eskf_exact as ee
import general_prior as gp
import scenes
from legkilo_b200 import Engine, abi, synth
import score_cases as sk

pytestmark = pytest.mark.gpu
CFG = abi.CONFIGS["leg_fusion"]


def _check(x, P, ex, what, x_in, P_in, k=None):
    ks = (ee.K_STEP, ee.K_POSE, ee.K_COV) if k is None else (k, k, k)
    return ee.check(x, P, ex, *ks, what=what, x_in=x_in, P_in=P_in)


# ---- lk_update_by_points ----------------------------------------------------------------------------------------------
GPU_SCENARIOS = ee.SCENARIOS + [("box", 256, "fixed", "dense", None), ("box", 40001, "wide", "dense", None)]


@pytest.mark.parametrize("sc", GPU_SCENARIOS, ids=ee.scenario_id)
def test_update_by_points_exact(sc):
    geometry, n, weight, prior, step = sc
    x, P, h, z, r = ee.case(geometry, n, weight, prior, 40 + n, step or (0.0,) * 6)
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(n))
    xg, Pg = Engine(CFG).update_by_points(x, P, h, z, r)
    _check(xg, Pg, ex, ee.scenario_id(sc), x, P)


def test_update_by_points_singular_is_a_zero_step():
    """Unit rows, R = 1, P66 = -I: I + A P66 is exactly zero in fp64, so the step is zero and x, P come back bit for bit."""
    x = ee.state(synth.rng(7)); P = -np.eye(30).ravel()
    h = np.eye(6); z = np.arange(1.0, 7.0); r = np.ones(6)
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(6))
    assert ex["zero"]
    xg, Pg = Engine(CFG).update_by_points(x, P, h, z, r)
    _check(xg, Pg, ex, "singular", x, P)


@pytest.mark.parametrize("side", [1 - 1e-6, 1 + 1e-6])
def test_update_by_points_step_at_the_exp_threshold(side):
    """A step whose attitude part is 1e-5 (1 -+ 1e-6): just inside and just outside so3_exp3's identity threshold. The
    exact step is linear in z, so z is scaled to put it there."""
    x, P, h, z, r = ee.case("box", 50, "fixed", "dense", 8)
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(50))
    nrm = float(np.linalg.norm([float(v) for v in ex["delta"][0:3]]))
    z = z * (ee.TH_EXP3 * side / nrm)
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(50))
    nrm = float(np.linalg.norm([float(v) for v in ex["delta"][0:3]]))
    assert abs(nrm / ee.TH_EXP3 - 1) > 1e-12 and (nrm > ee.TH_EXP3) == (side > 1)
    xg, Pg = Engine(CFG).update_by_points(x, P, h, z, r)
    _check(xg, Pg, ex, f"|dtheta| = {nrm!r}", x, P)


# ---- LiDAR buckets on the scan paths -----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _scene(name):
    if name == "plane":
        cfg, blob, pts = scenes.planar_scene(n=2048)
    elif name == "plane-45k":  # more than 40 000 points: a bucket sliced into many chunks
        cfg, blob, pts = scenes.planar_scene(n=45000)
    else:
        cfg, blob, scans = scenes.box_scene(batch=1)
        pts = scans[0]
    return cfg, blob, np.ascontiguousarray(pts, np.float32)


PATHS = {"batch-of-one": dict(fused=1, batch=1), "multi-kernel": dict(fused=0, batch=1), "batch-of-two": dict(fused=1, batch=2)}
# buckets: whole scans, the shortest prefix of the box scan with n_eff = 1 or 2 (the N == 1 rule reads the sum R lane of
# the cross-block reductions), and prefixes of 255 / 256 / 257 points (one chunk, one chunk full, a second chunk of one)
BUCKETS = ("box", "plane", "plane-45k", "box-neff1", "box-neff2", "box-pts255", "box-pts256", "box-pts257")
SCAN_CASES = [(p, b, q) for p in PATHS for b in BUCKETS for q in ("init", "dense")
              if not (b == "plane-45k" and p == "batch-of-one")]  # more than one chunk per block: never the batch-of-one kernel
SCAN_CASES += [(p, "box", q) for p in PATHS for q in ("asym", "scaled", "corr")]


def _scan_prior(kind, g, i):
    if i > 0:  # the second scan of a batch: its own dense prior
        return gp.dense_cov(g, scale=1.5)
    if kind == "init":
        return abi.init_cov(1)[0]
    if kind == "dense":
        return gp.dense_cov(g, scale=0.5)
    return ee.prior(kind, g).ravel()


def _bucket(eng, name, pts, x0, P0):
    """The points of bucket `name`, from the rows lk_debug_residuals finds at the first scan's prior."""
    if "-neff" in name:
        ok = np.flatnonzero(eng.debug_residuals(x0, P0, pts)["ok"])
        return pts[:ok[int(name.split("neff")[1]) - 1] + 1]
    if "-pts" in name:
        return pts[:int(name.split("pts")[1])]
    return pts


@pytest.mark.parametrize("path,bucket,prior", SCAN_CASES)
def test_scan_bucket_exact(path, bucket, prior):
    cfg, blob, pts = _scene(bucket.split("-")[0] if bucket != "plane-45k" else bucket)
    g = synth.rng(90)
    t = 5.0
    batch = PATHS[path]["batch"]
    x0 = np.concatenate([gp.moving_state(np.eye(3), (0.0, 0.0, 0.0)) for _ in range(batch)])
    P0 = np.stack([_scan_prior(prior, g, i) for i in range(batch)])
    clk = np.zeros(batch, abi.CLOCK_DTYPE); clk["last_predict_time"] = t; clk["last_update_time"] = t
    Q = abi.process_cov_Q(cfg)
    eng = Engine(cfg); eng.map_upload(blob)
    eng.set_param("fused", PATHS[path]["fused"])
    pts = _bucket(eng, bucket, pts, x0[:1], P0[0])
    n = len(pts)
    out = eng.scan_update(x0, P0, Q, clk, np.concatenate([pts] * batch), np.arange(batch + 1) * n, [t] * batch, iters=1)
    for i in range(batch):
        d = eng.debug_residuals(x0[i:i + 1], P0[i], pts)
        ok = d["ok"].astype(bool)
        assert int(ok.sum()) == int(out["n_eff"][i]) > 0, (int(ok.sum()), out["n_eff"])
        if bucket.startswith("box-neff") and i == 0:
            assert int(ok.sum()) == int(bucket.split("neff")[1])
        ex = ee.update_exact(x0[i:i + 1], P0[i], d["h"][ok], d["z"][ok], d["R"][ok], ee.depth_scan(int(ok.sum())))
        _check(out["x"][i:i + 1], out["P"][i], ex, f"{path} {bucket} {prior} scan {i} n_eff {int(ok.sum())}", x0[i:i + 1],
               P0[i])


# ---- lk_score_poses / lk_refine_poses ---------------------------------------------------------------------------------
def _sym(C):
    C = np.asarray(C, np.float64)
    return 0.5 * (C + C.T)


REFINE_COVS = {"narrow": (sk.ROT_COV, sk.POS_COV), "wide": (1e-2 * np.diag([1.0, 2.0, 3.0]), np.diag([0.3, 0.1, 0.2]))}
REFINE_CASES = [(b, pose, c) for b in ("box", "plane", "box-neff1", "box-neff2") for pose in ("at", "near") for c in REFINE_COVS]


@pytest.mark.parametrize("bucket,pose,covs", REFINE_CASES)
def test_score_and_refine_exact(bucket, pose, covs):
    """The record lk_score_poses returns at a pose against the exact sums of lk_debug_residuals' rows there (the count
    exactly), and one step of lk_refine_poses from it against the exact update restricted to the pose: P66 =
    blockdiag(rot_cov, pos_cov) (symmetric, as k_refine_step reads it), every other block of P zero."""
    cfg, blob, pts = _scene(bucket.split("-")[0])
    eng = Engine(cfg); eng.map_upload(blob)
    rc, pc = (_sym(c) for c in REFINE_COVS[covs])
    R0, p0 = (np.eye(3), np.zeros(3)) if pose == "at" else (synth.exp_so3((0.004, -0.006, 0.01)), np.array([0.03, -0.05, 0.02]))
    x0 = sk.pose_state(R0, p0)
    P = np.zeros((30, 30)); P[:3, :3] = rc; P[3:6, 3:6] = pc
    pts = _bucket(eng, bucket, pts, x0, sk.pose_cov(rc, pc))
    so = [0, len(pts)]
    rec = eng.score_poses(pts, so, [0], R0[None], p0[None], rc, pc)[0]
    d = eng.debug_residuals(x0, sk.pose_cov(rc, pc), pts)
    ok = d["ok"].astype(bool)
    n = int(ok.sum())
    assert int(rec[abi.SCORE_COUNT]) == rec[abi.SCORE_COUNT] == n > 0
    if bucket.startswith("box-neff"):
        assert n == int(bucket.split("neff")[1])
    exr, scale = ee.record_exact(d["h"][ok], d["z"][ok], d["R"][ok])
    assert (rec[abi.SCORE_SUM_Z2R + 1:] == 0).all()
    err = np.array([float(abs(ee.mp([rec[k]])[0] - exr[k])) for k in range(abi.SCORE_SUM_Z2R + 1)])
    q = ee._ratio(err, ee.gamma(ee.depth_scan(n) + 3) * scale)
    k = int(np.argmax(q))
    what = f"{bucket} pose {pose} covs {covs} n_eff {n}"
    print(f"eskf-exact record {what}: worst/scale {q[k]:.3g} at entry {k}")
    assert q[k] <= ee.K_STEP, (what, "record entry", k, err[k], scale[k])
    rot, pos, _ = eng.refine_poses(pts, so, [0], R0[None], p0[None], rc, pc, 1, want_records=False)
    ex = ee.update_exact(x0, P.ravel(), d["h"][ok], d["z"][ok], d["R"][ok], ee.depth_scan(n))
    e_att = ee.att_err(rot[0].ravel(), ex["R"])
    e_pos = np.array([float(abs(ee.mp([pos[0][j]])[0] - ex["rest"][j])) for j in range(3)])
    q_att = 0.0 if e_att == 0 else e_att / ex["d_att"]
    q_pos = float(ee._ratio(e_pos, ex["d_rest"][:3]).max())
    print(f"eskf-exact refine {what}: worst/scale position {q_pos:.3g} attitude {q_att:.3g} | cond(M) {ex['cond_M']:.2g}")
    assert q_pos <= ee.K_STEP and q_att <= ee.K_POSE, (what, q_pos, q_att)


# ---- inertial / kinematic observations ---------------------------------------------------------------------------------
def _sample(kind, contact):
    meas = (synth.imu_stream if kind == "imu" else synth.kinimu_stream)(1.0, 1.01)[:1].copy()
    if kind == "kin":
        meas["contact"][0] = contact
    return meas


def _predicted_cov(g, n=50):
    """dense_cov after 50 predicts of 5 ms, then its imu_a / imu_w standard deviations scaled up so that their variances
    are at least 1e4 times every pose variance (50 predicts alone reach 25x the attitude and 600x the position variances)."""
    x = gp.moving_state(np.eye(3), (1.0, 2.0, 0.5))
    P = gp.dense_cov(g).reshape(1, 900)
    xg, Pg = Engine(CFG).predict(x, P, abi.process_cov_Q(CFG), [0.005], True, True)
    for _ in range(n - 1):
        xg, Pg = Engine(CFG).predict(xg, Pg, abi.process_cov_Q(CFG), [0.005], True, True)
    P = Pg[0].reshape(30, 30)
    d = np.diag(P)
    sd = np.ones(30)
    sd[18:24] = np.sqrt(1e4 * d[:6].max() / d[18:24].min())
    P = P * np.outer(sd, sd)
    assert np.diag(P)[18:24].min() >= 1e4 * np.diag(P)[:6].max() * (1 - 1e-12)
    return P.ravel()


def _pivot_cov(cfg):
    """A P for which S = H P H^T + diag(r) of the inertial rows has S[0,0] = 0 exactly and cond(S) = 3: the
    elimination must swap rows."""
    r = np.array([cfg["imu_acc_meas_noise"]] * 2 + [cfg["imu_acc_z_meas_noise"]] + [cfg["imu_gyr_meas_noise"]] * 3)
    St = np.eye(6)[[1, 0, 2, 3, 4, 5]] + 0.5 * np.eye(6)[[0, 1, 3, 2, 5, 4]]
    St[0, 0] = 0.0
    P = 1e-2 * np.eye(30)
    P[9:15, 9:15] = St - np.diag(r)
    P[18:24, 18:24] = 0.0
    return P.ravel()


CONTACTS = {6: (0, 0, 0, 0), 9: (0, 1, 0, 0), 12: (2, 0, 0, -1), 15: (1, 1, 0, 1), 18: (1, 2, -1, 1)}


# the pivot prior is built for the inertial rows
OBS_CASES = [(m, q) for m in sorted(CONTACTS) for q in ("dense", "predicted", "tiny-kin-noise")] + [(6, "pivot")]


@pytest.mark.parametrize("m,prior", OBS_CASES)
def test_obs_exact(m, prior):
    kind = "imu" if m == 6 and prior != "tiny-kin-noise" else "kin"
    cfg = dict(CFG, kin_meas_noise=1e-12) if prior == "tiny-kin-noise" else CFG
    g = synth.rng(200 + m)
    x0 = gp.prior_at(gp.so3_uniform(g), (12.0, -7.5, 0.4), g)
    P0 = {"dense": lambda: gp.dense_cov(g), "predicted": lambda: _predicted_cov(g), "tiny-kin-noise": lambda: _predicted_cov(g),
          "pivot": lambda: _pivot_cov(cfg)}[prior]()
    meas = _sample(kind, CONTACTS[m])
    t = float(meas["stamp"][0])
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = t; clk["last_update_time"] = t
    Q = abi.process_cov_Q(cfg)
    eng = Engine(cfg)
    f = eng.obs_imu if kind == "imu" else eng.obs_kinimu
    xg, Pg, cg = f(x0, P0, Q, clk, meas, gravity=9.81, acc_norm=9.79)
    H, z, r, dH, dz = ee.obs_rows(x0, meas[0], cfg, 9.81, 9.79, kin=kind == "kin")
    assert H.rows == m
    ex = ee.dense_exact(x0, P0, H, z, r, dH, dz)
    _check(xg, Pg, ex, f"{kind} m {m} {prior}", x0, P0, k=ee.K_OBS)
    assert cg["last_predict_time"][0] == cg["last_update_time"][0] == t


# ---- predict ----------------------------------------------------------------------------------------------------------
PREDICT_DTS = (1e-9, 1e-4, 0.0123, 0.5, -0.005)  # |imu_w dt| 1.6e-10 (below 1e-7: Exp is the identity) ... 0.08


@pytest.mark.parametrize("mode", [(True, True), (True, False), (False, True), (False, False)], ids=str)
def test_predict_exact(mode):
    ps, pc = mode
    g = synth.rng(77)
    B = len(PREDICT_DTS)
    x0 = np.concatenate([gp.prior_at(gp.so3_uniform(g), g.uniform(-50.0, 50.0, 3), g) for _ in range(B)])
    P0 = []
    for i in range(B):
        P = gp.dense_cov(g).reshape(30, 30)
        sd = np.ones(30); sd[21:24] = 1e4  # imu_w variances 1e8 times the rest
        P0.append((P * np.outer(sd, sd)).ravel())
    P0 = np.stack(P0)
    Q = abi.process_cov_Q(CFG)
    xg, Pg = Engine(CFG).predict(x0, P0, Q, PREDICT_DTS, ps, pc)
    for i, dt in enumerate(PREDICT_DTS):
        ex = ee.predict_exact(x0[i:i + 1], P0[i], Q, dt, ps, pc)
        _check(xg[i:i + 1], Pg[i], ex, f"predict state {ps} cov {pc} dt {dt}", x0[i:i + 1], P0[i], k=ee.K_PRED)
