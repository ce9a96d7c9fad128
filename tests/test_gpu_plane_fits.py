"""Every plane fit the device map holds, from every producer, against the extended-precision init_plane
(tests/planefit_exact.py), with bounds scaled to each plane's conditioning: the bulk build, lk_first_frame, the three
streaming insert paths, lk_map_insert across a window boundary and fits that land in storage recycled by lk_map_slide.
Constructed voxels put warp_fit_plane (lk_plane.cuh) at its edges: point counts around the warp width and the 64-point
tile, l_min a hair either side of the threshold, eigen-gap edges, and degenerate voxels where the oracle's behaviour is
the reference."""
import numpy as np
import pytest

import lko
import map_insert_cases as mic
import planefit_exact as pe
import scenes
import test_gpu_map_memory as tmm
import test_planefit_exact as tpe
from first_frame_cases import load_first_frame
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
MAX_POINTS = list(tpe.MAX_POINTS)  # "default" (max_points_num 50) and "raised" (300: nothing freezes)
SAMPLE = 500  # leaves checked per map (seeded); the maps of constructed voxels are checked whole


def _engine(cfg, blob=None, **params):
    eng = Engine(cfg)
    for k, v in params.items():
        eng.set_param(k, v)
    if blob is not None:
        eng.map_upload(blob)
    return eng


def _build(cfg, pw, pb, R=None, rc=None, pc=None):
    eng = _engine(cfg)
    eng.map_build(pw, pb, R, rc, pc)
    return eng.map_download()


# ---- lk_map_build --------------------------------------------------------------------------------------------------------
OFFSETS = [(0.0, 0.0, 0.0), (1000.0, -700.0, 30.0), (1e4, -7e3, 30.0)]


def _scene(name, cfg, offset):
    if name == "planar":
        R, t = abi.extrinsics(cfg)
        pw, pb = synth.planar_map_points(half_extent=10.0, ext_R=R, ext_t=t)
        args = (pw, pb)
    elif name == "box":
        args = tpe._box(cfg, (0.0, 0.0, 0.0))
    else:
        args = tpe._cluttered()
    return ((args[0] + np.asarray(offset)).astype(np.float32),) + tuple(args[1:])


@pytest.mark.parametrize("mp", MAX_POINTS)
@pytest.mark.parametrize("offset", OFFSETS, ids=["origin", "1km", "10km"])
@pytest.mark.parametrize("scene", ["planar", "box", "cluttered"])
def test_map_build(scene, offset, mp):
    cfg = tpe._cfg("diter" if scene == "box" else "leg_fusion", mp)
    st = pe.check_map(_build(cfg, *_scene(scene, cfg, offset)), cfg, sample=SAMPLE, what=f"build {scene} {offset}")
    assert st["planes"] > 300


@pytest.mark.parametrize("mp", MAX_POINTS)
def test_map_build_voxel_0_4(mp):
    cfg = tpe._cfg("diter", mp, voxel_size=0.4)
    st = pe.check_map(_build(cfg, *_scene("box", cfg, (0.0, 0.0, 0.0))), cfg, sample=SAMPLE, what="build box v0.4")
    assert st["planes"] > 300


def test_map_build_max_layer_non_planes():
    """max_layer 1: the corner clusters leave fitted non-plane leaves at the max layer, which keep their points."""
    cfg = tpe._cfg("leg_fusion", "raised", max_layer=1)
    st = pe.check_map(_build(cfg, *_scene("cluttered", cfg, (0.0, 0.0, 0.0))), cfg, sample=SAMPLE, what="build max_layer 1")
    assert st["max_layer_non_planes"] > 5


# ---- lk_first_frame ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mp", MAX_POINTS)
@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_first_frame(kind, mp):
    cfg = tpe._cfg("leg_fusion", mp)
    d = load_first_frame(kind)
    eng = _engine(cfg)
    eng.first_frame(abi.default_states(1), d["raw0"], float(d["end0"]), gravity=9.81, world=False, **{kind: d["meas0"]})
    st = pe.check_map(eng.map_download(), cfg, sample=SAMPLE, what=f"first frame {kind}")
    assert st["planes"] > 300


# ---- lk_scan_update with update_map ----------------------------------------------------------------------------------------
INSERTS = {"two-launch": dict(fast_insert=1, fused_insert=0), "slice-and-sort": dict(fast_insert=0, fused_insert=0),
           "in-kernel": dict(fast_insert=1, fused_insert=1)}


@pytest.mark.parametrize("mp", MAX_POINTS)
@pytest.mark.parametrize("insert", list(INSERTS))
def test_scan_update_map(insert, mp):
    """Two streaming scans of one stream (test_gpu_map.py::_stream_case): leaves refitted every few insertions."""
    import test_gpu_parity as tp
    cfg0, blob, scans = scenes.box_scene(batch=2, streaming=True, stream0=700)
    cfg = tpe._cfg("leg_fusion", mp)
    eng = _engine(cfg, blob, **INSERTS[insert])
    x, P = tp._moving_state(), abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 9.99; clk["last_update_time"] = 9.985
    t0 = 10.0
    for s in scans:
        pts, offs, times = synth.bucketize(s, begin_time=t0)
        out = eng.scan_update(x, P, abi.process_cov_Q(cfg), clk, pts, [0, len(pts)], times, scan_bucket_ptr=[0, len(times)],
                              bucket_offsets=offs, iters=1, update_map=True)
        x, P, clk = out["x"], out["P"], out["clk"]
        t0 += 0.1
    blob1 = eng.map_download()
    _, _, _, aux, _ = abi.parse_map_blob(blob1)
    assert (aux["new_points"] > 0).any()  # leaves part-way to their next refit: the fitted prefix is what is checked
    st = pe.check_map(blob1, cfg, sample=SAMPLE, what=f"scan update {insert}")
    assert st["planes"] > 300


# ---- lk_map_insert -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mp", MAX_POINTS)
def test_map_insert_across_windows(mp):
    """Over two insert windows (lk_insert.cu: MAP_INSERT_WINDOW) on top of the box room's first-frame map."""
    import test_gpu_map_insert as tmi
    cfg = tpe._cfg("leg_fusion", mp)
    c = mic.room_trajectory(cfg, 48, 9700)
    assert len(c["pts"]) > 2 * tmi.WINDOW
    eng = _engine(cfg, mic.start_blob(cfg, c))
    eng.map_insert(*mic.call(c))
    st = pe.check_map(eng.map_download(), cfg, sample=SAMPLE, what="map insert")
    assert st["planes"] > 300


# ---- fits in recycled storage ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mp", MAX_POINTS)
def test_fits_in_recycled_storage(mp):
    """The floor of test_gpu_map_memory, sliding the window after every scan: once it is full, new roots take the nodes
    and tiles of the ones that slid out, and their fits land there."""
    cfg = dict(tmm.SLIDE_CFG)
    if tpe.MAX_POINTS[mp] is not None:
        cfg["max_points_num"] = tpe.MAX_POINTS[mp]
    s = tmm._Stream(cfg, oracle=False)
    recycled = 0
    for i in range(36):
        pos = (tmm.STEP_M * i, 0.0, 0.0)
        s.step(tmm._floor_scan(cfg, pos, i), pos=pos)
        before = s.eng.map_memory()
        s.eng.map_slide(pos)
        recycled = max(recycled, s.eng.map_memory()["free_nodes"] - before["free_nodes"])
    assert recycled > 0
    st = pe.check_map(s.eng.map_download(), cfg, sample=SAMPLE, what="after slides")
    assert st["planes"] > 300


# ---- constructed voxels --------------------------------------------------------------------------------------------------
def _frame(normal):
    n = np.asarray(normal, float) / np.linalg.norm(normal)
    a = np.cross(n, [0.0, 0.0, 1.0] if abs(n[2]) < 0.9 else [1.0, 0.0, 0.0])
    a /= np.linalg.norm(a)
    return a, np.cross(n, a), n


def _voxel(cell, vs, uv, w, normal):
    """Points q + u a + v b + w n in the root cell `cell` (q its centre), as float32."""
    q = (np.asarray(cell, float) + 0.5) * vs
    a, b, n = _frame(normal)
    return (q + uv[:, :1] * a + uv[:, 1:2] * b + w[:, None] * n).astype(np.float32)


class Voxels:
    """Constructed root voxels of one lk_map_build call: each in a cell of its own, with its float32 points."""

    def __init__(self, vs):
        self.vs, self.cells, self.pts, self.kind = vs, [], [], []

    def add(self, cell, pts, kind):
        assert np.all(np.floor(pts.astype(np.float64) / self.vs) == cell), (kind, cell)
        self.cells.append(tuple(cell)); self.pts.append(pts); self.kind.append(kind)

    def cloud(self):
        pw = np.concatenate(self.pts)
        pb = pw - np.float32([0.0, 0.0, -1.5])  # the body frame 1.5 m below: ranges of a few metres for calcBodyCov
        return pw, pb

    def roots(self, blob):
        _, roots, nodes, aux, pts = abi.parse_map_blob(blob)
        by_key = {tuple(int(k) for k in r["key"]): int(r["node"]) for r in roots}
        return [(by_key[c], nodes[by_key[c]], aux[by_key[c]]) for c in self.cells]


def _tilted_plane(g, n_pts, cell, vs, sigma=0.004, normal=None):
    """A plane through the voxel centre and (nearly) through the origin: d is tiny and |c| is not, so d's error is not
    hidden below one float ulp of d."""
    q = (np.asarray(cell, float) + 0.5) * vs
    if normal is None:
        r = g.standard_normal(3)
        normal = r - (r @ q) / (q @ q) * q
    uv = g.uniform(-0.45 * vs, 0.45 * vs, (n_pts, 2))
    return _voxel(cell, vs, uv, sigma * g.standard_normal(n_pts), normal)


def _counts_voxels(cfg, offset_cells):
    g = synth.rng(4100)
    vx = Voxels(cfg["voxel_size"])
    counts = [cfg["layer_init_num"][0] + 1, 31, 32, 33, 63, 64, 65, 128, 129]
    for j, n in enumerate(counts):
        vx.add(np.array([6 + 2 * j, 4, 1]) + offset_cells, _tilted_plane(g, n, np.array([6 + 2 * j, 4, 1]) + offset_cells,
                                                                         vx.vs), f"n={n}")
    return vx


@pytest.mark.parametrize("offset_cells", [(0, 0, 0), (200, -140, 6)], ids=["near", "100m"])
def test_point_counts_around_warp_and_tile(offset_cells):
    """layer_init_num + 1, 31..33, 63..65, 128, 129 points: warp sums with idle lanes, one and several 64-point tiles."""
    cfg = tpe._cfg("leg_fusion", "raised")
    vx = _counts_voxels(cfg, np.asarray(offset_cells))
    blob = _build(cfg, *vx.cloud())
    for (i, A, X), p, kind in zip(vx.roots(blob), vx.pts, vx.kind):
        assert int(X["pts_count"]) == len(p) and int(A["flags"]) & abi.NODE_IS_PLANE, kind
    st = pe.check_map(blob, cfg, what=f"point counts {offset_cells}")
    assert st["planes"] == len(vx.kind)


def _lmin(pts, thr):
    return pe.init_plane_exact(pts.astype(np.float64), np.zeros((len(pts), 6)), thr)["lam"][0]


def _near_threshold_voxel(g, cell, vs, thr32, target):
    """A slab whose exact l_min (of its float32 points) lands within a tenth of |target - thr32| of target: bisect the
    slab's half-thickness, then walk single-ulp steps of the points nearest the mid-plane, whose moves shift l_min the
    least."""
    n_pts = 96
    uv = g.choice([-1.0, 1.0], (n_pts, 2)) * g.uniform(0.15, 0.22, (n_pts, 2))  # in-plane variance ~0.035
    sgn = np.where(np.arange(n_pts) % 2 == 0, 1.0, -1.0)
    w0 = sgn * (1.0 + 0.05 * g.standard_normal(n_pts))
    w0[:8] = np.array([1e-2, -1e-2, 3e-3, -3e-3, 1e-3, -1e-3, 3e-4, -3e-4])  # tuning points near the mid-plane
    normal = np.r_[0.1 * g.standard_normal(2), 1.0]  # tilted a little: the slab stays inside its cell
    tol = 0.1 * abs(target - thr32)
    lo, hi = 0.5 * np.sqrt(target), 2.0 * np.sqrt(target)
    for _ in range(60):
        h = 0.5 * (lo + hi)
        pts = _voxel(cell, vs, uv, h * w0, normal)
        lam = _lmin(pts, thr32)
        if abs(lam - target) <= tol:
            return pts, lam
        lo, hi = (h, hi) if lam < target else (lo, h)
    _, _, n = _frame(normal)
    for j in range(8):
        axis = int(np.argmax(np.abs(n)))
        for _ in range(64):
            step = np.zeros_like(pts)
            step[j, axis] = np.spacing(pts[j, axis])
            lam_up = _lmin(pts + step, thr32)
            slope = lam_up - lam
            if slope == 0:
                break
            k = int(np.round((target - lam) / slope))
            if k == 0:
                break
            trial = pts.copy()
            trial[j, axis] = np.float32(pts[j, axis] + k * step[j, axis])
            lam_t = _lmin(trial, thr32)
            if abs(lam_t - target) >= abs(lam - target):
                break
            pts, lam = trial, lam_t
            if abs(lam - target) <= tol:
                return pts, lam
    return None


DECADES = [1e-3, 1e-4, 1e-5, 1e-6, 1e-7, 1e-8, 1e-9]


@pytest.fixture(scope="module")
def threshold_voxels():
    cfg = tpe._cfg("leg_fusion", "raised")
    thr32 = float(np.float32(cfg["min_eigen_value"]))
    g = synth.rng(4200)
    vx = Voxels(cfg["voxel_size"])
    j = 0
    for delta in DECADES:
        for s in (-1.0, 1.0):
            for tries in range(4):
                cell = np.array([2 + 2 * (j % 10), -12 + 2 * (j // 10), 0])
                j += 1
                r = _near_threshold_voxel(g, cell, vx.vs, thr32, thr32 * (1 + s * delta * (1 + g.uniform())))
                if r is not None:
                    vx.add(cell, r[0], (s, delta, r[1]))
                    break
    return cfg, vx


def test_is_plane_a_hair_either_side_of_the_threshold(threshold_voxels):
    """l_min = thr (1 +- d), d from 1e-3 down to 1e-9 (the decision band of these voxels is ~1e-13 relative): the device
    decides every one as the exact fit does. A non-plane root is cut, so its decision is read off its flags."""
    cfg, vx = threshold_voxels
    got = {(k[0], k[1]) for k in vx.kind}
    assert got == {(s, d) for d in DECADES for s in (-1.0, 1.0)}, sorted(got)
    blob = _build(cfg, *vx.cloud())
    for (i, A, X), p, (s, delta, lam) in zip(vx.roots(blob), vx.pts, vx.kind):
        ex = pe.init_plane_exact(p.astype(np.float64), np.zeros((len(p), 6)), cfg["min_eigen_value"])
        _, unit = pe.conditioning(ex)
        assert abs(ex["lam"][0] - ex["threshold"]) > pe.K_BAND * unit
        assert bool(int(A["flags"]) & abi.NODE_IS_PLANE) == ex["is_plane"] == (s < 0), (s, delta, lam, ex["threshold"])
    pe.check_map(blob, cfg, what="near threshold")


def test_eigen_gap_edges():
    """An exactly axis-aligned plane (diagonal covariance: eig_sym3 skips every rotation), a nearly isotropic in-plane
    spread (l_mid ~ l_max) and a nearly line-like voxel (small gap, large plane_var)."""
    cfg = tpe._cfg("leg_fusion", "raised")
    g = synth.rng(4300)
    vx = Voxels(cfg["voxel_size"])
    # dyadic lattice at z = 2.25: every moment exact, the covariance exactly diagonal
    lat = tpe._lattice(7, 5, 1, 0.0625, 0.03125, 1.0, (3.0 + 0.0625, 2.0 + 0.0625, 2.25)).astype(np.float32)
    vx.add((6, 4, 4), lat, "axis-aligned")
    ang = np.arange(72) * (2 * np.pi / 72)
    ring = np.c_[0.2 * np.cos(ang), 0.2 * np.sin(ang)] * (1 + 1e-4 * g.standard_normal((72, 1)))
    vx.add((10, 4, 2), _voxel((10, 4, 2), vx.vs, ring, 0.003 * g.standard_normal(72), (0.3, -0.4, 0.8)), "isotropic")
    line = np.c_[g.uniform(-0.22, 0.22, 80), 0.004 * g.standard_normal(80)]
    vx.add((14, 4, 2), _voxel((14, 4, 2), vx.vs, line, 0.003 * g.standard_normal(80), (0.5, 0.2, -0.7)), "line-like")
    blob = _build(cfg, *vx.cloud())
    st = pe.check_map(blob, cfg, what="eigen-gap edges")
    assert st["planes"] == 3
    (_, A, _), = vx.roots(blob)[:1]
    np.testing.assert_array_equal(np.abs(A["normal"]), [0.0, 0.0, 1.0])
    fits = [pe.init_plane_exact(p.astype(np.float64), np.zeros((len(p), 6)), 0.01) for p in vx.pts]
    assert fits[1]["lam"][2] - fits[1]["lam"][1] < 1e-2 * fits[1]["lam"][2]
    assert fits[2]["gap"] < 1e-3 * fits[2]["lam"][2]


def test_degenerate_voxels_follow_the_oracle():
    """Exactly collinear and coincident points: no meaningful exact fit, so the oracle's behaviour is the reference: the
    same decision, the record finite where the oracle's is, and a scan through the voxels gives the oracle's n_eff."""
    cfg = dict(abi.CONFIGS["leg_fusion"])
    R, t = abi.extrinsics(cfg)
    pw, pb = synth.planar_map_points(half_extent=6.0, ext_R=R, ext_t=t)
    vx = Voxels(cfg["voxel_size"])
    xs = np.float32(0.25) + np.arange(40, dtype=np.float32) * np.float32(0.005)
    vx.add((4, 2, 0), np.c_[2.0 + xs, np.full(40, 1.125), np.full(40, 0.375)].astype(np.float32), "collinear-axis")
    vx.add((6, 2, 0), np.c_[3.0 + xs, 1.0 + xs, np.full(40, 0.25)].astype(np.float32), "collinear-diagonal")
    vx.add((8, 2, 0), np.tile(np.float32([[4.2, 1.3, 0.3]]), (30, 1)), "coincident")
    vx.add((10, 2, 0), np.tile(np.float32([[5.1, 1.1, 0.1]]), (6, 1)), "coincident-min")
    dw, db = vx.cloud()
    pw2, pb2 = np.concatenate([pw, dw]), np.concatenate([pb, db])
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw2, pb2)
    eng = _engine(cfg)
    eng.map_build(pw2, pb2)
    ob, db_ = o.map_export(), eng.map_download()
    for (io, Ao, _), (idv, Ad, _), kind in zip(vx.roots(ob), vx.roots(db_), vx.kind):
        assert (int(Ao["flags"]) & 0xff07) == (int(Ad["flags"]) & 0xff07), (kind, hex(int(Ao["flags"])), hex(int(Ad["flags"])))
        if int(Ao["flags"]) & abi.NODE_IS_PLANE:
            for k in ("center", "normal", "plane_var", "d", "radius"):
                np.testing.assert_array_equal(np.isfinite(Ad[k]), np.isfinite(Ao[k]), err_msg=f"{kind} {k}")
    # a scan that reaches every degenerate voxel, against the map each side built
    g = synth.rng(4400)
    scan_w = np.concatenate([p[g.integers(0, len(p), 12)] + 0.01 * g.standard_normal((12, 3)) for p in vx.pts])
    floor = synth.planar_scan(n=1024, ext_R=R, ext_t=t, stream=3, rotvec=(0.0, 0.0, 0.0), trans=(0.0, 0.0, 0.0))
    scan_b = synth.world_to_body(scan_w.astype(np.float64), np.eye(3), np.zeros(3), R, t)
    pts = np.concatenate([floor, np.c_[scan_b, np.zeros(len(scan_b))].astype(np.float32)])
    x0, P0, Q = abi.default_states(1), abi.init_cov(1), abi.process_cov_Q(cfg)
    clk = np.zeros(1, abi.CLOCK_DTYPE)
    out = eng.scan_update(x0, P0, Q, clk, pts, [0, len(pts)], [0.0], iters=1)
    o.set_filter(x0, P0, Q, clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    ro = o.predict_update_point(0.0, pts)
    assert int(out["n_eff"][0]) == ro["n_eff"], (int(out["n_eff"][0]), ro["n_eff"])
