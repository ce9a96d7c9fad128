"""Pins tests/eskf_exact.py without a device: its results do not move with the working precision, equal closed forms
(one row, a diagonal system, the literal Kalman gain of Woodbury's identity), and its scales behave as error scales. Then
holds the CPU oracle against it on the scenarios of tests/test_gpu_filter_exact.py and prints the oracle's worst ratios,
which say whether the device is more or less accurate than the CPU restatement of the reference."""
import mpmath
import numpy as np
import pytest

import eskf_exact as ee
import lko
from legkilo_b200 import abi, synth

CFG = abi.CONFIGS["leg_fusion"]
# The oracle's bound, in the helper's units with its own summation depth (n, one serial sum): worst measured 0.89. Its
# literal gain is another form (K = P H^T (H P H^T + R)^-1), so only its information form is held to it; the literal
# one is printed (it reaches 1.7e4 on the step where A P66 ~ 1e10).
K_ORACLE = 4.0


def _rel(a, b):
    return float(max(abs(x - y) for x, y in zip(a, b)) / max(max(abs(x) for x in b), mpmath.mpf(1e-300)))


def test_digits_agree():
    x, P, h, z, r = ee.case("box", 300, "wide", "dense", 1)
    a = ee.update_exact(x, P, h, z, r, ee.depth_rows(300), dps=40)
    b = ee.update_exact(x, P, h, z, r, ee.depth_rows(300), dps=60)
    with mpmath.workdps(60):
        assert _rel(list(a["delta"]), list(b["delta"])) < 1e-35
        assert _rel(list(a["P"]), list(b["P"])) < 1e-35
        assert _rel(list(a["R"]), list(b["R"])) < 1e-35
    for k in ("d_delta", "dP"):
        np.testing.assert_allclose(a[k], b[k], rtol=1e-12)


def test_single_row_closed_form():
    """One row: delta = P6 h^T z s / (R + s h P66 h^T), P - P6 h^T h P[0:6,:] s / (R + s h P66 h^T), s = R / (R + 1e-4)."""
    x, P, h, z, r = ee.case("box", 1, "fixed", "dense", 2, step=(0.1, 0, 0, 0, 0.2, 0))
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(1))
    with mpmath.workdps(ee.DPS):
        Pm = ee.mp(P.reshape(30, 30)); hm = ee.mp(h)  # 1 x 6
        R = mpmath.mpf(float(r[0])); s = R / (R + mpmath.mpf(1e-4))
        den = R + s * (hm * Pm[0:6, 0:6] * hm.T)[0, 0]
        delta = Pm[:, 0:6] * hm.T * (s * float(z[0]) / den)
        Pn = Pm - Pm[:, 0:6] * hm.T * hm * Pm[0:6, :] * (s / den)
        assert _rel(list(ex["delta"]), list(delta)) < 1e-35
        assert _rel(list(ex["P"]), list(Pn)) < 1e-35


def test_diagonal_closed_form():
    """Rows along the axes and a diagonal P66: y_k = b_k / (1 + A_kk P_kk)."""
    g = synth.rng(3)
    n = 24
    h = np.zeros((n, 6)); h[np.arange(n), np.arange(n) % 6] = g.uniform(0.5, 2.0, n)
    r = g.uniform(1e-3, 1e-2, n); z = g.standard_normal(n)
    P = np.diag(g.uniform(1e-4, 1.0, 30))
    ex = ee.update_exact(abi.default_states(1), P.ravel(), h, z, r, ee.depth_rows(n))
    with mpmath.workdps(ee.DPS):
        for k in range(6):
            sel = np.arange(n) % 6 == k
            A = mpmath.fsum(mpmath.mpf(float(v)) ** 2 / float(w) for v, w in zip(h[sel, k], r[sel]))
            b = mpmath.fsum(mpmath.mpf(float(v)) * float(q) / float(w) for v, q, w in zip(h[sel, k], z[sel], r[sel]))
            y = b / (1 + A * float(P[k, k]))
            assert abs(ex["delta"][k] - float(P[k, k]) * y) <= 1e-35 * abs(float(P[k, k]) * y)


@pytest.mark.parametrize("n", [2, 5, 6, 18])
def test_woodbury(n):
    """The information form equals the literal gain K = P H^T (H P H^T + R)^-1 at 40 digits."""
    x, P, h, z, r = ee.case("corridor", n, "wide", "dense", 10 + n)
    ex = ee.update_exact(x, P, h, z, r, ee.depth_rows(n))
    with mpmath.workdps(ee.DPS):
        Pm = ee.mp(P.reshape(30, 30)); H = ee.mp(h)
        S = H * Pm[0:6, 0:6] * H.T
        for k in range(n):
            S[k, k] += float(r[k])
        K = Pm[:, 0:6] * H.T * mpmath.inverse(S)
        delta = K * ee.mp(z)
        Pn = Pm - K * H * Pm[0:6, :]
        assert _rel(list(ex["delta"]), list(delta)) < 1e-33
        assert _rel(list(ex["P"]), list(Pn)) < 1e-33


def test_scales_follow_a_rigid_frame_change():
    """Rows expressed in a frame turned by a signed permutation (an exact rigid rotation): every scale is the same
    scale, permuted."""
    x, P, h, z, r = ee.case("box", 40, "fixed", "dense", 5)
    Q = np.eye(3)[[2, 0, 1]] * np.array([1.0, -1.0, 1.0])[:, None]
    T = np.eye(30); T[:3, :3] = Q; T[3:6, 3:6] = Q
    P30 = P.reshape(30, 30)
    a = ee.update_exact(x, P, h, z, r, ee.depth_rows(40))
    b = ee.update_exact(x, (T.T @ P30 @ T).ravel(), h @ T[:6, :6], z, r, ee.depth_rows(40))
    np.testing.assert_allclose(b["d_delta"], np.abs(T.T) @ a["d_delta"], rtol=1e-12)
    np.testing.assert_allclose(b["dP"], np.abs(T.T) @ a["dP"] @ np.abs(T), rtol=1e-12)
    assert abs(b["d_att"] - a["d_att"]) <= 1e-12 * a["d_att"]


def test_scales_grow_with_conditioning():
    """The same rows against a prior scaled up by 10^k: cond(M) grows, and the step's bound relative to the step grows
    with it, by at least a hundredth of cond(M)'s growth."""
    x, P, h, z, r = ee.case("box", 50, "fixed", "dense", 6)
    P30 = P.reshape(30, 30)
    last, first = 0.0, None
    for k in range(0, 11, 2):
        Pk = P30.copy(); Pk[:6, :6] *= 10.0 ** k
        ex = ee.update_exact(x, Pk.ravel(), h, z, r, ee.depth_rows(50))
        d = np.array([float(v) for v in ex["delta"]])[:6]
        rel = float((ex["d_delta"][:6] / np.abs(d).max()).max())
        assert rel > last, (k, rel, last, ex["cond_M"])
        first = first or (rel, ex["cond_M"])
        last = rel
    assert last / first[0] > 1e-2 * ex["cond_M"] / first[1], (first, last, ex["cond_M"])


# ---- the oracle against the helper ------------------------------------------------------------------------------------
@pytest.mark.parametrize("sc", ee.SCENARIOS, ids=ee.scenario_id)
def test_oracle_update_by_points(sc):
    geometry, n, weight, prior, step = sc
    x, P, h, z, r = ee.case(geometry, n, weight, prior, 40 + n, step or (0.0,) * 6)
    ex = ee.update_exact(x, P, h, z, r, n + 13)
    for mode in (lko.GAIN_INFORMATION, lko.GAIN_LITERAL):
        o = lko.Oracle(CFG); o.set_filter(x, P, None, None)
        o.update_by_points(h, z, r, gain_mode=mode)
        xo, Po, _, _ = o.get_filter()
        k = K_ORACLE if mode == lko.GAIN_INFORMATION else np.inf
        ee.check(xo, Po, ex, k, k, k, f"oracle {'information' if mode else 'literal'} {ee.scenario_id(sc)}", x_in=x, P_in=P)


def test_oracle_singular_system():
    """Unit rows, R = 1, P66 = -I: I + A P66 is exactly zero. The helper (as the device, lk_solve.cuh) takes a zero step;
    the oracle's LU, like the reference's, divides by the zero pivot, so the device's rule has no fp64 counterpart to
    match and tests/test_gpu_filter_exact.py holds it to x and P returned bit for bit."""
    x = ee.state(synth.rng(7)); P = -np.eye(30)
    h = np.eye(6); z = np.arange(1.0, 7.0); r = np.ones(6)
    ex = ee.update_exact(x, P.ravel(), h, z, r, ee.depth_rows(6))
    assert ex["zero"]
    o = lko.Oracle(CFG); o.set_filter(x, P.ravel(), None, None)
    o.update_by_points(h, z, r, gain_mode=lko.GAIN_INFORMATION)
    xo, Po, _, _ = o.get_filter()
    assert not np.isfinite(Po).all() and not np.isfinite(ee._x36(xo)).all()


@pytest.mark.parametrize("kind,contact", [("imu", None), ("kin", (0, 0, 0, 0)), ("kin", (0, 1, 0, 0)), ("kin", (2, 0, 0, -1)),
                                          ("kin", (1, 1, 0, 1)), ("kin", (1, 2, -1, 1))])
def test_oracle_obs(kind, contact):
    """obs_imu / obs_kinimu with one sample at the clock (both predicts are no-ops), m = 6 ... 18."""
    import general_prior as gp
    for noise in (CFG["kin_meas_noise"], 1e-12):
        cfg = dict(CFG, kin_meas_noise=noise)
        g = synth.rng(300)
        x0 = gp.prior_at(gp.so3_uniform(g), (12.0, -7.5, 0.4), g)
        P0 = gp.dense_cov(g)
        meas = (synth.imu_stream if kind == "imu" else synth.kinimu_stream)(1.0, 1.01)[:1].copy()
        if kind == "kin":
            meas["contact"][0] = contact
        t = float(meas["stamp"][0])
        clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = t; clk["last_update_time"] = t
        o = lko.Oracle(cfg); o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk)
        o.set_options(imu_mode_only=kind == "imu", gravity=9.81, acc_norm=9.79)
        (o.obs_imu if kind == "imu" else o.obs_kinimu)(meas)
        xo, Po, _, _ = o.get_filter()
        H, z, r, dH, dz = ee.obs_rows(x0, meas[0], cfg, 9.81, 9.79, kin=kind == "kin")
        ex = ee.dense_exact(x0, P0, H, z, r, dH, dz)
        ee.check(xo, Po, ex, K_ORACLE, K_ORACLE, K_ORACLE, f"oracle {kind} m {H.rows} kin_meas_noise {noise}")


@pytest.mark.parametrize("dt", [1e-9, 1e-4, 0.0123, 0.5, -0.005])
def test_oracle_predict(dt):
    import general_prior as gp
    g = synth.rng(77)
    x0 = gp.prior_at(gp.so3_uniform(g), g.uniform(-50.0, 50.0, 3), g)
    sd = np.ones(30); sd[21:24] = 1e4
    P0 = (gp.dense_cov(g).reshape(30, 30) * np.outer(sd, sd)).ravel()
    Q = abi.process_cov_Q(CFG)
    for ps, pc in ((True, True), (True, False), (False, True)):
        o = lko.Oracle(CFG); o.set_filter(x0, P0, Q, None); o.predict(dt, ps, pc)
        xo, Po, _, _ = o.get_filter()
        ex = ee.predict_exact(x0, P0, Q, dt, ps, pc)
        ee.check(xo, Po, ex, K_ORACLE, K_ORACLE, K_ORACLE, f"oracle predict state {ps} cov {pc} dt {dt}")


@pytest.mark.parametrize("prior", ["init", "dense"])
def test_oracle_predict_update_point(prior):
    """A bucket stamped at the clock through the oracle's predictUpdatePoint, against the exact update of its own rows."""
    import general_prior as gp
    import scenes
    cfg, blob, pts = scenes.planar_scene(n=2048)
    x0 = gp.moving_state(np.eye(3), (0.0, 0.0, 0.0))
    P0 = abi.init_cov(1)[0] if prior == "init" else gp.dense_cov(synth.rng(90), scale=0.5)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 5.0; clk["last_update_time"] = 5.0
    o = lko.Oracle(cfg); o.map_import(blob); o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    ro = o.predict_update_point(5.0, pts, debug=True)
    ok = ro["ok"].astype(bool)
    assert int(ok.sum()) == ro["n_eff"] > 0
    xo, Po, _, _ = o.get_filter()
    ex = ee.update_exact(x0, P0, ro["h"][ok], ro["z"][ok], ro["R"][ok], int(ok.sum()) + 13)
    ee.check(xo, Po, ex, K_ORACLE, K_ORACLE, K_ORACLE, f"oracle predict_update_point {prior}")
