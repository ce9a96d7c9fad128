"""The extended-precision init_plane (tests/planefit_exact.py) pinned on closed forms, and the CPU oracle's plane fits
held against it: how far the one-pass formula of voxel_map.cc:49-54 actually lands from the exact fit, per plane, in
units of that plane's conditioning."""
import mpmath
import numpy as np
import pytest

import lko
import planefit_exact as pe
import scenes
from legkilo_b200 import abi, synth

THR = 0.01


def _lattice(mx, my, mz, hx, hy, hz, origin):
    g = np.stack(np.meshgrid(np.arange(mx) * hx, np.arange(my) * hy, np.arange(mz) * hz, indexing="ij"), -1).reshape(-1, 3)
    return g + np.asarray(origin, np.float64)


def _vars(n, seed=3):
    g = synth.rng(seed)
    A = g.standard_normal((n, 3, 3)) * 1e-2
    return A @ A.transpose(0, 2, 1) + 1e-5 * np.eye(3)


def _plane_var_direct(pw, var, lam, e, imin):
    """voxel_map.cc:74-92 term by term in float64, given the eigen-decomposition."""
    n = len(pw)
    c = pw.mean(0)
    out = np.zeros((6, 6))
    for p, S in zip(pw, var):
        F = np.zeros((3, 3))
        for m in range(3):
            if m != imin:
                F[m] = (p - c) / (n * (lam[imin] - lam[m])) @ (np.outer(e[:, m], e[:, imin]) + np.outer(e[:, imin], e[:, m]))
        J = np.vstack([e @ F, np.eye(3) / n])
        out += J @ S @ J.T
    return out


def test_axis_aligned_lattice_closed_form():
    """Uniform lattices: centre and covariance in closed form (variance of m equal steps h: h^2 (m^2 - 1) / 12), the
    eigenvectors the axes, and plane_var the reference formula evaluated on them."""
    mx, my, mz, hx, hy, hz = 7, 5, 2, 0.0625, 0.03125, 0.0078125
    pw = _lattice(mx, my, mz, hx, hy, hz, (1024.0, -512.0, 32.0))
    var = _vars(len(pw))
    ex = pe.init_plane_exact(pw, var, THR)
    lam = [h * h * (m * m - 1) / 12 for m, h in ((mz, hz), (my, hy), (mx, hx))]
    np.testing.assert_array_equal(np.asarray(ex["lam"]), lam)
    np.testing.assert_array_equal(ex["center"].astype(np.float64),
                                  [1024.0 + hx * (mx - 1) / 2, -512.0 + hy * (my - 1) / 2, 32.0 + hz * (mz - 1) / 2])
    np.testing.assert_array_equal(ex["normal"].astype(np.float64), [0.0, 0.0, 1.0])
    assert ex["is_plane"] and ex["radius"] == pytest.approx(np.sqrt(lam[2]), rel=1e-15)
    assert ex["d"] == -ex["center"][2]
    e = np.eye(3)
    pv = _plane_var_direct(pw, var, [lam[2], lam[1], lam[0]], e, 2)
    np.testing.assert_allclose(ex["plane_var"].astype(np.float64), pv, rtol=0, atol=1e-13 * np.abs(pv).max())


def test_invariant_under_a_rigid_motion():
    """A signed axis permutation and a translation, both exact in float64: the fit moves with the points, to the last
    digit carried; a general rotation moves it up to the rounding of the rotated points."""
    g = synth.rng(11)
    pw = np.round(np.c_[g.uniform(0, 0.5, (60, 2)), 0.01 * g.standard_normal(60)] * 4096) / 4096
    var = _vars(len(pw), 5)
    R = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, 1.0], [-1.0, 0.0, 0.0]])
    t = np.array([2048.0, -256.0, 64.0])
    a = pe.init_plane_exact(pw, var, THR)
    b = pe.init_plane_exact(pw @ R.T + t, R @ var @ R.T, THR)
    np.testing.assert_allclose(np.asarray(b["lam"]), np.asarray(a["lam"]), rtol=1e-30)
    na = R @ a["normal"]
    sgn = np.sign(float(na @ b["normal"]))
    np.testing.assert_allclose((sgn * na).astype(np.float64), b["normal"].astype(np.float64), rtol=0, atol=1e-18)
    np.testing.assert_allclose(b["center"].astype(np.float64), R @ a["center"].astype(np.float64) + t, rtol=0, atol=1e-12)
    T = np.zeros((6, 6)); T[:3, :3] = sgn * R; T[3:, 3:] = R
    Va = T @ a["plane_var"].astype(np.float64) @ T.T
    np.testing.assert_allclose(b["plane_var"].astype(np.float64), Va, rtol=0, atol=1e-15 * np.abs(Va).max())
    # general rotation: the rotated points are rounded to float64
    Rg = synth.exp_so3([0.3, -0.2, 0.9])
    c = pe.init_plane_exact(pw @ Rg.T + t, Rg @ var @ Rg.T, THR)
    nc = Rg @ a["normal"].astype(np.float64)
    nc *= np.sign(nc @ c["normal"].astype(np.float64))
    np.testing.assert_allclose(c["normal"].astype(np.float64), nc, rtol=0, atol=1e-9)
    np.testing.assert_allclose(np.asarray(c["lam"]), np.asarray(a["lam"]), rtol=1e-9)


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (1000.0, -700.0, 30.0), (1e4, 1e4, -50.0)])
def test_forty_digits_agree_with_sixty(offset):
    g = synth.rng(21)
    pw = np.c_[g.uniform(0, 0.5, (80, 2)), 0.003 * g.standard_normal(80)] @ synth.exp_so3([0.4, 0.1, -0.3]).T + offset
    var = _vars(len(pw), 7)
    a = pe.init_plane_exact(pw, var, THR, dps=40)
    b = pe.init_plane_exact(pw, var, THR, dps=60)
    for k in ("center", "normal"):
        np.testing.assert_allclose(a[k], b[k], rtol=2e-18, atol=0)
    np.testing.assert_allclose(np.asarray(a["lam"]), np.asarray(b["lam"]), rtol=1e-30)
    np.testing.assert_allclose(a["plane_var"], b["plane_var"], rtol=0, atol=1e-17 * float(np.abs(b["plane_var"]).max()))
    assert a["is_plane"] == b["is_plane"] and a["d"] == b["d"] and a["radius"] == b["radius"]


def test_exact_decision_uses_the_float_threshold():
    """planer_threshold_ is a float: l_min between float(0.01) and 0.01 is not a plane."""
    thr32 = float(np.float32(THR))
    assert thr32 < THR
    g = synth.rng(5)
    xy = g.uniform(-0.5, 0.5, (100, 2))
    base = np.r_[np.c_[xy, np.ones(100)], np.c_[xy, -np.ones(100)]]  # z uncorrelated with x, y: l_min = var(z)
    for target, want in ((0.5 * (THR + thr32), False), (thr32 * (1 + 1e-9), False), (thr32 * (1 - 1e-9), True)):
        pw = base * [1.0, 1.0, np.sqrt(target)]
        ex = pe.init_plane_exact(pw, _vars(len(pw)), THR)
        assert abs(ex["lam"][0] - target) < 1e-12 * target and ex["is_plane"] == want, (ex["lam"], target)


# ---- the oracle's own distance from exact ------------------------------------------------------------------------------
def _oracle_build(cfg, pw, pb, R=None, rc=None, pc=None):
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw, pb, R, rc, pc)
    return o.map_export()


def _box(cfg, offset):
    R, t = abi.extrinsics(cfg)
    pw, pb = synth.BoxScene(ground_half_extent=18.0).map_points(ext_R=R, ext_t=t)
    return (pw + np.asarray(offset)).astype(np.float32), pb


def _cluttered():
    """The clutter of test_gpu_map.py::test_build_cluttered_scene_subdivides, plus clusters at the corners of a 0.25 m
    lattice: a layer-1 octant (0.25 m) of a 0.5 m voxel holds pieces of its eight corner clusters, so its l_min is
    above 0.01 and it is cut again, down to layer 2 (or stays a non-plane leaf when max_layer is 1)."""
    g = synth.rng(77)
    n = 60000
    pw = np.concatenate([
        g.uniform(-4, 4, (n // 2, 3)),
        np.c_[g.uniform(-4, 4, (n // 4, 2)), 0.13 + 0.002 * g.standard_normal(n // 4)],
        g.uniform(4, 6, (n // 4, 3)) * np.array([1, 1, 0.05]),
        -6.0 - 0.25 * g.integers(0, 5, (n // 4, 3)) + g.uniform(-0.03, 0.03, (n // 4, 3))]).astype(np.float32)
    pb = pw.copy()
    pb[:, 2] -= 0.2
    return pw, pb, synth.exp_so3([0.01, -0.02, 0.03]), np.diag([1e-6, 2e-6, 3e-6]), np.diag([4e-6, 5e-6, 6e-6])


MAX_POINTS = {"default": None, "raised": 300}  # raised: nothing freezes, so every leaf keeps the points it was fitted on


def _cfg(name, mp, **kw):
    cfg = dict(abi.CONFIGS[name], **kw)
    if MAX_POINTS[mp] is not None:
        cfg["max_points_num"] = MAX_POINTS[mp]
    return cfg


@pytest.mark.parametrize("mp", list(MAX_POINTS))
@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (1000.0, -700.0, 30.0)])
def test_oracle_box_room(offset, mp):
    cfg = _cfg("diter", mp)
    st = pe.check_map(_oracle_build(cfg, *_box(cfg, offset)), cfg, sample=600, what=f"oracle box {offset}")
    assert st["planes"] > 500


@pytest.mark.parametrize("max_layer", [2, 1])
@pytest.mark.parametrize("mp", list(MAX_POINTS))
def test_oracle_cluttered_scene(mp, max_layer):
    """Roots cut to layer 2: fitted leaves at every layer; with max_layer 1, non-plane leaves at the max layer."""
    cfg = _cfg("leg_fusion", mp, max_layer=max_layer)
    st = pe.check_map(_oracle_build(cfg, *_cluttered()), cfg, sample=600, what=f"oracle cluttered max_layer {max_layer}")
    assert st["planes"] > 100 and st["layers"] == set(range(max_layer + 1))
    assert (st["max_layer_non_planes"] > 10) == (max_layer == 1)


def test_oracle_voxel_size_0_4():
    cfg = _cfg("diter", "raised", voxel_size=0.4)
    st = pe.check_map(_oracle_build(cfg, *_box(cfg, (0.0, 0.0, 0.0))), cfg, sample=600, what="oracle box v0.4")
    assert st["planes"] > 500


@pytest.mark.parametrize("mp", list(MAX_POINTS))
def test_oracle_streaming_update_map(mp):
    """Two streaming scans with UpdateVoxelMap: leaves refitted every few points, new roots and octants on demand."""
    cfg0, blob, scans = scenes.box_scene(batch=2, streaming=True, stream0=700)
    cfg = _cfg("leg_fusion", mp)
    o = lko.Oracle(cfg)
    o.map_import(blob)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 9.99; clk["last_update_time"] = 9.985
    o.set_filter(abi.default_states(1), abi.init_cov(1), abi.process_cov_Q(cfg), clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=True)
    t0 = 10.0
    for s in scans:
        pts, _, _ = synth.bucketize(s, begin_time=t0)
        o.process_scan(t0, pts)
        t0 += 0.1
    st = pe.check_map(o.map_export(), cfg, sample=600, what="oracle streaming")
    assert st["planes"] > 300


def test_oracle_init_plane_matches_at_its_conditioning():
    """lko.init_plane on single voxels from the origin to 10 km: within the same per-plane bounds the maps are held to."""
    g = synth.rng(31)
    worst = dict(normal=0.0, var=0.0)
    for off in (0.0, 30.0, 1e3, 1e4):
        for k in range(6):
            n = int(g.integers(6, 200))
            R = synth.exp_so3(g.standard_normal(3))
            pw = (np.c_[g.uniform(0, 0.5, (n, 2)), 0.02 * g.standard_normal(n)] @ R.T + off * g.standard_normal(3))
            pw = pw.astype(np.float32).astype(np.float64)
            var = _vars(n, k)
            ex = pe.init_plane_exact(pw, var, THR)
            orc = lko.init_plane(pw, var.reshape(n, 9), THR)
            assert orc["is_plane"] == ex["is_plane"]
            if not ex["is_plane"]:
                continue
            scale, _ = pe.conditioning(ex)
            no = orc["normal"] * np.sign(orc["normal"] @ ex["normal"].astype(np.float64))
            worst["normal"] = max(worst["normal"], float(np.abs(no - ex["normal"]).max()) / scale)
            # plane_var's cross blocks follow the normal's sign
            V = orc["plane_var"].copy()
            if orc["normal"] @ ex["normal"].astype(np.float64) < 0:
                V[:3, 3:] *= -1; V[3:, :3] *= -1
            worst["var"] = max(worst["var"], float(np.abs(V - ex["plane_var"]).max() / np.abs(ex["plane_var"]).max()) / scale)
    print(f"oracle init_plane worst/eps-scale: normal {worst['normal']:.3g} plane_var {worst['var']:.3g}")
    assert worst["normal"] <= pe.K_NORMAL and worst["var"] <= pe.K_VAR
    assert mpmath.mp.dps == 15  # the helper leaves mpmath's global precision alone
