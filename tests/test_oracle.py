"""CPU pins of the oracle (the C++ restatement) — the reference ships no golden vectors, so the pins
are self-made (SURVEY.md §8c): (1) literal N x N gain vs 6 x 6 information form, (2) an independent
numpy / LAPACK mirror, (3) analytic cases, (4) committed golden fixtures."""
import os

import numpy as np
import pytest

import lko
import np_mirror as npm
import scenes
from legkilo_b200 import abi, synth

CFG = abi.CONFIGS["leg_fusion"]
G = synth.rng(4242)


def _state_from(x):
    return x["rot"][0].reshape(3, 3).copy(), x["pos"][0].copy()


# ---- math_utils.hpp ----------------------------------------------------------------------------
def test_exp_log_thresholds_and_roundtrip():
    for v in ([0.3, -0.2, 0.5], [1e-3, 2e-3, -1e-3], [2e-5, 0, 0]):
        np.testing.assert_allclose(lko.exp3(v), npm.exp3(v), atol=1e-15)
        np.testing.assert_allclose(lko.log_so3(lko.exp3(v)), v, rtol=1e-6, atol=1e-12)
    # Exp(v1,v2,v3) returns I at or below 1e-5 rad (math_utils.hpp:58): sub-10-urad corrections vanish
    assert np.array_equal(lko.exp3([9e-6, 0, 0]), np.eye(3))
    assert not np.array_equal(lko.exp3([1.1e-5, 0, 0]), np.eye(3))


def test_boxplus_boxminus_roundtrip():
    x = abi.default_states(1)
    x["rot"][0] = lko.exp3([0.1, -0.2, 0.3]).ravel()
    d = G.normal(size=30) * 1e-2
    y = lko.boxplus(x, d)
    np.testing.assert_allclose(lko.boxminus(y, x), d, rtol=1e-6, atol=1e-12)


# ---- calcBodyCov (voxel_map.cc:22-40) -------------------------------------------------------------
@pytest.mark.parametrize("pb", [[3.0, -1.0, 0.5], [0.2, 0.1, 7.0], [5.0, 2.0, 0.0], [-12.0, 4.0, -0.7]])
def test_calc_body_cov_vs_mirror_and_closed_form(pb):
    cov, pb2 = lko.calc_body_cov(pb, 0.04, 0.2)
    cov_m, pb_m = npm.calc_body_cov(pb, 0.04, 0.2)
    np.testing.assert_allclose(cov, cov_m, rtol=1e-12, atol=1e-18)
    assert pb2[2] == (1e-4 if pb[2] == 0 else pb[2])  # the z == 0 mutation (:23)
    # closed form used by the CUDA kernels: rv u u^T + range^2 dv (I - u u^T)
    u = pb2 / np.linalg.norm(pb2)
    rng = float(np.float32(np.linalg.norm(pb2)))
    rv = float(np.float32(0.04) * np.float32(0.04))
    dv = np.sin(float(np.float32(0.2)) * 0.017453293) ** 2
    closed = rv * np.outer(u, u) + rng * rng * dv * (np.eye(3) - np.outer(u, u))
    np.testing.assert_allclose(cov, closed, rtol=1e-12, atol=1e-18)


# ---- init_plane (voxel_map.cc:42-117) ---------------------------------------------------------------
def _plane_points(n, normal, offset, spread=0.2, noise=0.005, seed=1):
    g = synth.rng(seed)
    normal = np.asarray(normal, float) / np.linalg.norm(normal)
    a = np.cross(normal, [0.3, 0.5, 0.8]); a /= np.linalg.norm(a)
    b = np.cross(normal, a)
    uv = g.uniform(-spread, spread, (n, 2))
    pw = offset + uv[:, :1] * a + uv[:, 1:] * b + noise * g.standard_normal((n, 1)) * normal
    var = np.array([np.diag(g.uniform(1e-4, 4e-4, 3)) + 1e-5 * np.ones((3, 3)) for _ in range(n)])
    return pw, var


@pytest.mark.parametrize("n,normal,offset", [(8, [0, 0, 1], [3.0, 4.0, -0.75]), (30, [1, 2, 0.5], [-80.0, 45.0, 2.0]),
                                            (50, [0.1, 1.0, 0.0], [150.0, -90.0, 1.0])])
def test_init_plane_vs_mirror(n, normal, offset):
    pw, var = _plane_points(n, normal, np.asarray(offset))
    a = lko.init_plane(pw, var.reshape(n, 9))
    b = npm.init_plane(pw, var)
    assert a["is_plane"] and b["is_plane"]
    sgn = np.sign(a["normal"] @ b["normal"])
    np.testing.assert_allclose(a["center"], b["center"], rtol=1e-13)
    np.testing.assert_allclose(a["normal"], sgn * b["normal"], atol=1e-8)
    pv_b = b["plane_var"].copy()
    if sgn < 0:
        pv_b[:3, 3:] *= -1; pv_b[3:, :3] *= -1
    np.testing.assert_allclose(a["plane_var"], pv_b, rtol=1e-5, atol=1e-7 * np.abs(pv_b).max())
    assert abs(a["d"] - sgn * float(b["d"])) <= 1e-5 * max(1, abs(a["d"]))
    assert abs(a["radius"] - float(b["radius"])) <= 1e-6
    # plane covariance is symmetric PSD up to rounding
    np.testing.assert_allclose(a["plane_var"], a["plane_var"].T, atol=1e-12 * np.abs(a["plane_var"]).max())
    assert np.linalg.eigvalsh(0.5 * (a["plane_var"] + a["plane_var"].T)).min() > -1e-12 * np.abs(a["plane_var"]).max()


def test_init_plane_rejects_volume():
    pw = synth.rng(5).uniform(-0.25, 0.25, (40, 3)) + [5, 5, 5]  # variance 0.021 > min_eigen_value 0.01
    var = np.tile(np.eye(3).ravel() * 1e-4, (40, 1))
    assert not lko.init_plane(pw, var)["is_plane"]


# ---- residual rows (voxel_map.cc:363-427, KILO.cc:122-210) vs mirror -----------------------------------
def test_bucket_rows_vs_numpy_mirror():
    cfg, blob, _ = scenes.planar_scene(n=16, half_extent=8.0)
    Rx, tx = abi.extrinsics(cfg)
    pts = synth.planar_scan(n=200, radius=7.0, ext_R=Rx, ext_t=tx, stream=12)
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    x0["rot"][0] = lko.exp3([1e-3, -2e-3, 5e-4]).ravel(); x0["pos"][0] = (0.01, 0.02, -0.01)
    o = lko.Oracle(cfg); o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE)); o.set_options(update_map=False)
    r = o.predict_update_point(0.0, pts, debug=True)
    _, roots, nodes, aux, mpts = abi.parse_map_blob(blob)
    keymap = {tuple(k["key"]): int(k["node"]) for k in roots}
    R, p = _state_from(x0); Re, te = abi.extrinsics(cfg); P = P0.reshape(30, 30)
    checked = 0
    for i, q in enumerate(pts):
        pb = q[:3].astype(np.float64)
        pi = Re @ pb + te; pw = R @ pi + p
        bcov, _ = npm.calc_body_cov(pb, cfg["dept_err"], cfg["beam_err"])
        var = npm.point_var(R, Re, te, bcov, pi, P)
        loc = (pw / cfg["voxel_size"]).astype(np.float32)
        loc = np.where(loc < 0, (loc.astype(np.float64) - 1.0).astype(np.float32), loc)
        key = tuple(int(v) for v in loc.astype(np.int32))  # truncation
        assert key == tuple(r["key"][i])
        if key not in keymap:
            assert not r["ok"][i]; continue
        nd = nodes[keymap[key]]
        assert nd["flags"] & 1
        pvm = np.zeros((6, 6)); pvm[np.triu_indices(6)] = nd["plane_var"]; pvm = pvm + np.triu(pvm, 1).T
        plane = dict(normal=nd["normal"], center=nd["center"], d=nd["d"], radius=nd["radius"], plane_var=pvm)
        res = npm.plane_residual(pw, var, plane, cfg["sigma_num"])
        if res is None:
            continue  # the oracle may still succeed through the neighbour voxel
        assert r["ok"][i]
        h, z, Rk = npm.obs_row(R, Re, pi, bcov, plane, pw, res, cfg["lidar_point_meas_ratio"])
        np.testing.assert_allclose(r["h"][i], h, rtol=1e-9, atol=1e-12)
        assert r["z"][i] == z
        np.testing.assert_allclose(r["R"][i], Rk, rtol=1e-9)
        checked += 1
    assert checked > 150


# ---- updateByPoints (eskf.cc:91-113) -----------------------------------------------------------------
def _random_filter(seed):
    g = synth.rng(seed)
    A = g.standard_normal((30, 30)) * 1e-3
    P = A @ A.T + 1e-6 * np.eye(30)
    x = abi.default_states(1)
    x["rot"][0] = lko.exp3(g.normal(size=3) * 0.1).ravel(); x["pos"][0] = g.normal(size=3)
    return x, P


@pytest.mark.parametrize("n", [1, 2, 7, 300])
def test_update_by_points_literal_vs_information_vs_mirror(n):
    g = synth.rng(100 + n)
    x0, P0 = _random_filter(n)
    h = g.standard_normal((n, 6)); z = g.standard_normal(n) * 1e-2; r = g.uniform(1e-3, 1e-2, n)
    res = []
    for mode in (lko.GAIN_LITERAL, lko.GAIN_INFORMATION):
        o = lko.Oracle(CFG); o.set_filter(x0, P0.ravel(), None, None)
        o.update_by_points(h, z, r, gain_mode=mode)
        x, P, _, _ = o.get_filter()
        res.append((lko.boxminus(x, x0), P.reshape(30, 30)))
    d_m, P_m = npm.update_by_points_literal(P0, h, z, r)
    # Exp's 1e-5 identity threshold acts on delta_theta; compare what survives it
    for d, P in res:
        dd = d_m.copy()
        if np.linalg.norm(dd[:3]) <= 1e-5:
            dd[:3] = 0
        np.testing.assert_allclose(d, dd, rtol=1e-7, atol=1e-10 * np.abs(dd).max())
        np.testing.assert_allclose(P, P_m, rtol=1e-7, atol=1e-10 * np.abs(P_m).max())
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=1e-8, atol=1e-12 * np.abs(res[0][0]).max())
    np.testing.assert_allclose(res[0][1], res[1][1], rtol=1e-8, atol=1e-12 * np.abs(res[0][1]).max())


def test_config1_literal_pin_2048_points():
    """BASELINE config 1 on the CPU: 2 048-pt planar scan, identity prior, 1 iteration, the
    reference's literal N x N measurement-space form vs the information form the device uses."""
    cfg, blob, pts = scenes.planar_scene()
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    out = []
    for mode in (lko.GAIN_LITERAL, lko.GAIN_INFORMATION):
        o = lko.Oracle(cfg); o.map_import(blob)
        o.set_filter(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE)); o.set_options(gain_mode=mode, update_map=False)
        r = o.predict_update_point(0.0, pts)
        x, P, _, _ = o.get_filter()
        out.append((r["n_eff"], x, P))
    assert out[0][0] == out[1][0] > 0.9 * len(pts)
    scenes.check_filter(out[1][1], out[1][2], out[0][1], out[0][2], 8e-13, 7e-13)  # measured 8.4e-15 sd, 8.0e-15
    # the filter moved towards the true pose (Exp([2,-1,3]e-3), [0.02,-0.01,0.03]) where the plane constrains it
    d = lko.boxminus(out[0][1], x0)
    assert 1.2e-3 < d[0] < 2.2e-3 and -1.2e-3 < d[1] < -0.6e-3 and d[5] > 0


def test_filter_comparison_catches_pose_block_errors():
    """scenes.state_err / cov_err at the tolerances of the device's streaming tests, on the oracle's output for the inputs
    of test_gpu_parity.py::test_streaming_buckets_static_map. There ~50 predicts make the imu_w / imu_a variances ~1e4
    times the pose block's, which an error measured against P's largest entry cannot see past."""
    import test_gpu_parity as tp
    cfg, blob, scans = scenes.box_scene(batch=1, streaming=True, stream0=500)
    pts, _, _ = synth.bucketize(scans[0], begin_time=100.0)
    x0 = tp._moving_state(); P0 = abi.init_cov(1)
    clk0 = np.zeros(1, abi.CLOCK_DTYPE); clk0["last_predict_time"] = 99.99; clk0["last_update_time"] = 99.985
    runs = {}
    for gain in (lko.GAIN_LITERAL, lko.GAIN_INFORMATION):
        _, x, P, _, _ = tp._oracle_stream(cfg, blob, pts, 100.0, x0, P0, clk0, gain=gain)
        runs[gain] = x, P.reshape(30, 30)
    x, P = runs[lko.GAIN_INFORMATION]
    assert np.abs(P).max() > 1e3 * np.abs(P[:6, :6]).max()
    assert scenes.state_err(x, x, P) == 0.0 and scenes.cov_err(P, P) == 0.0
    # the literal and the information form differ in arithmetic only
    scenes.check_filter(*runs[lko.GAIN_LITERAL], x, P, tp.STATE_TOL, tp.COV_TOL)
    bad = P.copy(); bad[:6, :6] *= 1.1  # the whole pose block of P 10 % off
    e_block = scenes.cov_err(bad, P)
    bad = P.copy(); bad[:3, 3:6] = 0.0; bad[3:6, :3] = 0.0  # attitude-position cross block dropped
    e_cross = scenes.cov_err(bad, P)
    step = lko.boxminus(x, x0)
    e_step = scenes.state_err(lko.boxplus(x, np.r_[0.01 * step[:3], np.zeros(27)]), x, P)  # attitude step 1 % off
    print(f"pose block x 1.1: {e_block!r}; cross block zeroed: {e_cross!r}; attitude step + 1 %: {e_step!r} sd")
    assert e_block > tp.COV_TOL and e_cross > tp.COV_TOL and e_step > tp.STATE_TOL


def test_noise_free_plane_gives_zero_innovation():
    cfg = CFG; R, t = abi.extrinsics(cfg)
    pw, pb = synth.planar_map_points(half_extent=6.0, sigma=0.0, ext_R=R, ext_t=t)
    o = lko.Oracle(cfg); o.build_voxel_map(pw, pb)
    pts = synth.planar_scan(n=400, radius=5.0, sigma=0.0, rotvec=(0, 0, 0), trans=(0, 0, 0), ext_R=R, ext_t=t)
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    o.set_filter(x0, P0, None, np.zeros(1, abi.CLOCK_DTYPE)); o.set_options(update_map=False)
    r = o.predict_update_point(0.0, pts, debug=True)
    x, P, _, _ = o.get_filter()
    assert r["n_eff"] > 300 and np.abs(r["z"]).max() < 1e-6
    assert np.abs(lko.boxminus(x, x0)).max() < 1e-7
    P = P.reshape(30, 30)
    assert P[5, 5] < 0.95e-6 and abs(P[3, 3] - 1e-6) < 1e-9  # z observed by a horizontal plane, x not


# ---- predict (eskf.cc:64-89) ------------------------------------------------------------------------
def test_predict_vs_mirror_and_dt0_is_exact_noop():
    x0, P0 = _random_filter(9)
    x0["imu_w"][0] = (0.05, -0.02, 0.3); x0["imu_a"][0] = (0.2, -0.1, 9.6); x0["vel"][0] = (1.0, 0.5, -0.2)
    Q = abi.process_cov_Q(CFG)
    o = lko.Oracle(CFG); o.set_filter(x0, P0.ravel(), Q, None)
    o.predict(0.013, False, True)
    _, P1, _, _ = o.get_filter()
    R, _ = _state_from(x0)
    F = npm.fx(R, x0["imu_a"][0], x0["imu_w"][0], 0.013)
    np.testing.assert_allclose(P1.reshape(30, 30), F @ P0 @ F.T + 0.013 ** 2 * Q.reshape(30, 30), rtol=1e-12, atol=1e-18)
    o.predict(0.013, True, False)
    x1, _, _, _ = o.get_filter()
    d = lko.boxminus(x1, x0)
    np.testing.assert_allclose(d[3:6], 0.013 * x0["vel"][0], rtol=1e-12)
    np.testing.assert_allclose(d[6:9], 0.013 * (R @ x0["imu_a"][0] + x0["grav"][0]), rtol=1e-12)
    o2 = lko.Oracle(CFG); o2.set_filter(x0, P0.ravel(), Q, None)
    o2.predict(0.0, True, True)
    x2, P2, _, _ = o2.get_filter()
    assert np.array_equal(P2, P0.ravel()) and x2.tobytes() == x0.tobytes()


# ---- IMU / Kin+IMU observations (KILO.cc:235-314, eskf.cc:125-145) ----------------------------------------
def test_imu_and_kinimu_updates_vs_mirror():
    x0, P0 = _random_filter(21)
    x0["imu_w"][0] = (0.05, -0.02, 0.3); x0["imu_a"][0] = (0.2, -0.1, 9.6); x0["vel"][0] = (0.3, 0.1, 0.0)
    Q = abi.process_cov_Q(CFG)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 5.0; clk["last_update_time"] = 5.0
    imu = np.zeros(1, abi.IMU_DTYPE); imu["stamp"] = 5.0; imu["acc"] = (0.1, 0.2, 9.7); imu["gyr"] = (0.04, -0.01, 0.28)
    o = lko.Oracle(CFG); o.set_filter(x0, P0.ravel(), Q, clk); o.set_options(gravity=9.81, acc_norm=9.81)
    o.obs_imu(imu)   # dt = 0: pure update; (gravity / acc_norm) = 1 (KILO.cc:247)
    x1, P1, _, c1 = o.get_filter()
    z = np.concatenate([imu["acc"][0] - x0["imu_a"][0] - x0["ba"][0], imu["gyr"][0] - x0["imu_w"][0] - x0["bw"][0]])
    r = np.array([CFG["imu_acc_meas_noise"]] * 2 + [CFG["imu_acc_z_meas_noise"]] + [CFG["imu_gyr_meas_noise"]] * 3)
    d_m, P_m = npm.update_by_imu(P0, z, r)
    np.testing.assert_allclose(lko.boxminus(x1, x0), d_m, rtol=1e-8, atol=1e-12)
    np.testing.assert_allclose(P1.reshape(30, 30), P_m, rtol=1e-8, atol=1e-14)
    assert c1["last_update_time"][0] == 5.0
    kin = np.zeros(1, abi.KINIMU_DTYPE); kin["stamp"] = 5.0; kin["acc"] = imu["acc"]; kin["gyr"] = imu["gyr"]
    kin["contact"][0] = (1, 0, 1, 0)
    kin["foot_pos"][0] = [[0.2, -0.1, -0.3], [0.2, 0.1, -0.3], [-0.2, -0.1, -0.3], [-0.2, 0.1, -0.3]]
    kin["foot_vel"][0] = [[0.01, 0.0, 0.02], [0, 0, 0], [-0.02, 0.01, 0.0], [0, 0, 0]]
    o = lko.Oracle(CFG); o.set_filter(x0, P0.ravel(), Q, clk); o.set_options(imu_mode_only=False, gravity=9.81, acc_norm=9.81)
    o.obs_kinimu(kin)
    x2, P2, _, _ = o.get_filter()
    R, _ = _state_from(x0); w = x0["imu_w"][0]
    H = np.zeros((12, 30)); H[:6, 9:15] = np.eye(6); H[:6, 18:24] = np.eye(6)
    zz = list(z); rr = list(r)
    for k, leg in enumerate((0, 2)):
        fp, fv = kin["foot_pos"][0][leg], kin["foot_vel"][0][leg]
        wpv = npm.skew(w) @ fp + fv
        H[6 + 3 * k:9 + 3 * k, 0:3] = -R @ npm.skew(wpv); H[6 + 3 * k:9 + 3 * k, 6:9] = np.eye(3)
        H[6 + 3 * k:9 + 3 * k, 21:24] = -R @ npm.skew(fp)
        zz += list(-x0["vel"][0] - R @ wpv); rr += [CFG["kin_meas_noise"]] * 3
    d_m, P_m = npm.update_by_kinimu(P0, H, np.array(zz), np.array(rr))
    np.testing.assert_allclose(lko.boxminus(x2, x0), d_m, rtol=1e-7, atol=1e-12)
    np.testing.assert_allclose(P2.reshape(30, 30), P_m, rtol=1e-7, atol=1e-13)


# ---- octree state machine (voxel_map.cc:119-241) --------------------------------------------------------
def test_octree_refit_and_freeze_rules():
    cfg = CFG; R, t = abi.extrinsics(cfg)
    pw, var = _plane_points(80, [0, 0, 1], np.array([0.25, 0.25, 0.25]), spread=0.2, noise=0.002, seed=3)
    pw = pw.astype(np.float32)
    o = lko.Oracle(cfg)
    def stats():
        _, roots, nodes, aux, _ = abi.parse_map_blob(o.map_export())
        return nodes[0], aux[0]
    o.build_voxel_map(pw[:5], pw[:5] - t.astype(np.float32))      # 5 points: below the init threshold (> 5)
    n, a = stats(); assert not (n["flags"] & 2) and a["pts_count"] == 5 and a["new_points"] == 5
    o2 = lko.Oracle(cfg); o2.build_voxel_map(pw[:6], pw[:6] - t.astype(np.float32))
    _, _, nodes, aux, _ = abi.parse_map_blob(o2.map_export())
    assert nodes[0]["flags"] & 1 and nodes[0]["flags"] & 2 and aux[0]["pts_count"] == 6 and aux[0]["new_points"] == 0
    o3 = lko.Oracle(cfg); o3.build_voxel_map(pw[:60], pw[:60] - t.astype(np.float32))   # > 50: frozen at once
    _, _, nodes, aux, _ = abi.parse_map_blob(o3.map_export())
    assert nodes[0]["flags"] & 1 and not (nodes[0]["flags"] & 4) and aux[0]["pts_count"] == 0


def test_map_export_import_roundtrip():
    import mapcmp
    g = synth.rng(77)
    pw = np.concatenate([g.uniform(-2, 2, (6000, 3)), np.c_[g.uniform(-2, 2, (3000, 2)), 0.13 + 0.002 * g.standard_normal(3000)]]).astype(np.float32)
    pb = pw.copy(); pb[:, 2] -= 0.2
    o1 = lko.Oracle(CFG); o1.build_voxel_map(pw, pb)
    blob = o1.map_export()
    o = lko.Oracle(CFG); o.map_import(blob)
    st = mapcmp.compare_blobs(blob, o.map_export(), rtol=1e-15)
    assert st["planes"] > 50 and st["interior"] > 50


# ---- golden fixtures --------------------------------------------------------------------------------------
def test_golden_config1():
    """tests/golden/config1_planar.npz (made by tests/golden/make_golden.py from this oracle): pins the
    oracle, the scene generator and the map blob format against silent drift."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_planar.npz"))
    cfg, blob, pts = scenes.planar_scene()
    assert np.array_equal(pts, g["pts"])
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    o = lko.Oracle(cfg); o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE)); o.set_options(gain_mode=lko.GAIN_LITERAL, update_map=False)
    r = o.predict_update_point(0.0, pts)
    x, P, _, _ = o.get_filter()
    assert r["n_eff"] == int(g["n_eff"])
    np.testing.assert_allclose(x.view(np.float64), g["x"], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(P, g["P"], rtol=1e-9, atol=1e-18)
