"""lk_score_poses on the device: its records against the reference's counts (tests/golden/ref_score_poses.npz), against
lk_debug_residuals' rows at the same pose, against the staged-copies composition it replaces (n_effective of
lk_batch_run(iters=1)); bitwise invariance to the other poses of the call; ragged sets; nothing else on the handle moves;
the errors; and the search recipe of INTEGRATION.md §5 end to end."""
import ctypes as C

import numpy as np
import pytest

import lko
import score_cases as sk
import scenes
import test_gpu_map_images as mi
from legkilo_b200 import Engine, abi, lib, synth

pytestmark = pytest.mark.gpu
# Sums against float64 sums of the same rows (score_cases.record_err: each entry in units of the sum of its terms'
# absolute values), 100x the worst measured on an H100 80GB HBM3 (700 W): 1.2e-14 against lk_debug_residuals (hilti),
# 2.2e-15 against the oracle's rows of the fixture (whose R may differ from the device's by the rounding of the collapsed
# sigma_plane)
DEBUG_TOL = 1.2e-12
FIXTURE_TOL = 2.2e-13


def _score(eng, pts, rot, pos, set_offsets=None, pose_set=None, rot_cov=sk.ROT_COV, pos_cov=sk.POS_COV):
    so = [0, len(pts)] if set_offsets is None else set_offsets
    ps = np.zeros(len(rot), np.uint32) if pose_set is None else pose_set
    return eng.score_poses(pts, so, ps, rot, pos, rot_cov, pos_cov)


def _debug_record(eng, pts, R, p):
    d = eng.debug_residuals(sk.pose_state(R, p), sk.pose_cov()[None], pts)
    return sk.row_record(d["ok"], d["h"], d["z"], d["R"]), d


def _near_poses(R0, p0, stream):
    g = synth.rng(stream)
    rots, poss = [R0], [np.asarray(p0, float)]
    for rs, ts in ((0.003, 0.01), (0.01, 0.05), (0.03, 0.1), (0.1, 0.3), (0.2, 0.8)):
        rots.append(synth.exp_so3(g.normal(0.0, rs, 3)) @ R0)
        poss.append(np.asarray(p0, float) + g.normal(0.0, ts, 3))
    return np.array(rots), np.array(poss)


# ---- the reference's counts ------------------------------------------------------------------------------------------
def test_fixture_counts_equal_reference():
    d = sk.load_fixture()
    eng = Engine(abi.CONFIGS["leg_fusion"])
    eng.map_upload(d["blob"])
    rec = _score(eng, d["pts"], d["rot"], d["pos"], rot_cov=d["rot_cov"], pos_cov=d["pos_cov"])
    np.testing.assert_array_equal(rec[:, abi.SCORE_COUNT].astype(np.int64), d["counts"])
    err = max(sk.record_err(rec[i], d["oracle_record"][i], d["oracle_scale"][i]) for i in range(len(rec)))
    print(f"[score] fixture: worst record error {err:.3g}")
    assert err <= FIXTURE_TOL


# ---- against lk_debug_residuals at the same pose ---------------------------------------------------------------------
def _scene(name):
    if name in ("leg_fusion", "hilti"):
        cfg, blob, scans = scenes.box_scene(name)
        eng = Engine(cfg)
        eng.map_upload(blob)
        return eng, cfg, scans[0]
    if name == "voxel_0.4":  # a voxel size that is no power of two: the key divides
        cfg = dict(abi.CONFIGS["leg_fusion"], voxel_size=0.4)
        R, t = abi.extrinsics(cfg)
        sc = synth.BoxScene(ground_half_extent=10.0, wall=7.3, voxel=0.4)
        pw, pb = sc.map_points(ext_R=R, ext_t=t)
        o = lko.Oracle(cfg)
        o.build_voxel_map(pw, pb)
        eng = Engine(cfg)
        eng.map_upload(o.map_export())
        pts = sc.scan(rotvec=(0.002, -0.001, 0.003), trans=(0.01, -0.02, 0.01), ext_R=R, ext_t=t, blind=cfg["blind"], stream=905,
                      **synth.VLP16)
        return eng, cfg, pts
    # the shelf of test_gpu_map_images.test_bulk_build_box_room: roots cut into octants whose planes only a descent finds
    cfg = abi.CONFIGS["diter"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=18.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    rs = synth.rng(804)
    n = 40 * 8 * 8 * 2
    shelf = np.c_[rs.uniform(2.0, 6.0, (n, 2)), np.where(np.arange(n) % 2 == 0, 0.125, 0.375) + 0.005 * rs.standard_normal(n)]
    eng = Engine(cfg)
    eng.map_build(np.concatenate([pw, shelf.astype(np.float32)]), np.concatenate([pb, mi._body_pts(cfg, shelf)[:, :3]]))
    kids = mi._child_planes(eng.map_download())
    pts = np.concatenate([mi._room_scan(cfg, sc, 801), mi._body_pts(cfg, mi._on_planes(eng.map_download(), kids, 3, synth.rng(802)))])
    return eng, cfg, pts


@pytest.mark.parametrize("name", ["leg_fusion", "hilti", "voxel_0.4", "descent"])
def test_records_match_debug_rows(name):
    eng, cfg, pts = _scene(name)
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 910)
    rec = _score(eng, pts, rot, pos)
    worst, descent = 0.0, 0
    for i in range(len(rot)):
        (ref, scale), d = _debug_record(eng, pts, rot[i], pos[i])
        assert int(rec[i, abi.SCORE_COUNT]) == int(d["ok"].sum()), i
        worst = max(worst, sk.record_err(rec[i], ref, scale))
        assert (rec[i, 30:] == 0).all()
        if name == "descent":
            home = mi._root_flags(eng.map_download(), d["key"])
            descent += int((d["ok"].astype(bool) & (home >= 0) & ((home & abi.NODE_IS_PLANE) == 0)).sum())
    print(f"[score] {name}: worst record error against the debug rows {worst:.3g}, counts {rec[:, abi.SCORE_COUNT].tolist()}")
    assert worst <= DEBUG_TOL
    assert rec[0, abi.SCORE_COUNT] > 0.5 * len(pts)
    if name == "descent":
        assert descent > 1000, descent


# ---- against the staged-copies composition ---------------------------------------------------------------------------
def test_counts_equal_batch_composition():
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    pts = scans[0]
    eng = Engine(cfg)
    eng.map_upload(blob)
    rot, pos = sk.grid_poses(np.eye(3), np.zeros(3), np.linspace(-0.3, 0.3, 4), synth.rng(920).uniform(-1.0, 1.0, (16, 3)))
    rec = _score(eng, pts, rot, pos)
    M, n = len(rot), len(pts)
    x = np.concatenate([sk.pose_state(rot[i], pos[i]) for i in range(M)])
    P = np.tile(sk.pose_cov(), (M, 1))
    eng.stage(x, P, abi.process_cov_Q(cfg), np.zeros(M, abi.CLOCK_DTYPE), np.tile(pts, (M, 1)), np.arange(M + 1) * n, np.zeros(M))
    eng.run(iters=1)
    out = eng.fetch(want_world=False)
    np.testing.assert_array_equal(out["n_eff"].astype(np.int64), rec[:, abi.SCORE_COUNT].astype(np.int64))
    assert len(set(out["n_eff"].tolist())) > 10


# ---- invariance ------------------------------------------------------------------------------------------------------
def test_record_does_not_depend_on_the_other_poses():
    """4 096 poses of one 28 800-point scan (113 chunks: the poses run in two windows), against each pose scored alone,
    the call in reversed order, and a second run: bitwise."""
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    pts = scans[0]
    assert len(pts) > 28000
    eng = Engine(cfg)
    eng.map_upload(blob)
    off = np.stack(np.meshgrid(np.linspace(-1, 1, 16), np.linspace(-1, 1, 16), [0.0], indexing="ij"), -1).reshape(-1, 3)
    rot, pos = sk.grid_poses(np.eye(3), np.zeros(3), np.linspace(-0.2, 0.2, 16), off)
    assert len(rot) == 4096
    rec = _score(eng, pts, rot, pos)
    assert rec[:, abi.SCORE_COUNT].min() > 0
    rev = _score(eng, pts, rot[::-1], pos[::-1])[::-1]
    assert rev.tobytes() == rec.tobytes()
    assert _score(eng, pts, rot, pos).tobytes() == rec.tobytes()
    rows_per_pose = (len(pts) + 255) // 256
    boundary = ((1 << 18) // (16 * rows_per_pose)) * 16  # first pose of the second window
    for i in (0, 1, 15, 16, 2047, boundary - 1, boundary, 4095):
        assert _score(eng, pts, rot[i:i + 1], pos[i:i + 1]).tobytes() == rec[i:i + 1].tobytes(), i
    # the same poses mixed into another call: a subset, interleaved with a second set
    idx = np.array([4095, 7, boundary, 3, boundary - 1])
    so = [0, len(pts), 2 * len(pts)]
    mix = _score(eng, np.concatenate([pts, pts[::-1]]), np.repeat(rot[idx], 2, 0), np.repeat(pos[idx], 2, 0), so,
                 np.tile([0, 1], len(idx)).astype(np.uint32))
    assert mix[0::2].tobytes() == rec[idx].tobytes()


# ---- shapes ----------------------------------------------------------------------------------------------------------
def test_ragged_sets():
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    pts = scans[0]
    eng = Engine(cfg)
    eng.map_upload(blob)
    sizes = [300, 0, 1, 2000, 255, 257, 5000]
    so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    sets = np.concatenate([pts[::3][:sum(sizes)]])
    assert len(sets) == sum(sizes)
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 930)
    rot = np.concatenate([rot] * 6); pos = np.concatenate([pos] * 6)
    pos[-3:] += 1000.0  # outside the map
    ps = (np.arange(len(rot)) % 7).astype(np.uint32)
    rec = _score(eng, sets, rot, pos, so, ps)
    for m in range(len(rot)):
        s = int(ps[m])
        alone = _score(eng, sets[so[s]:so[s + 1]], rot[m:m + 1], pos[m:m + 1])
        assert alone.tobytes() == rec[m:m + 1].tobytes(), m
        if sizes[s] == 0 or m >= len(rot) - 3:
            assert (rec[m] == 0).all(), m
        elif sizes[s] > 200 and m % 6 < 3:  # the three poses nearest the truth
            assert rec[m, abi.SCORE_COUNT] > 0, m
    one = [m for m in range(len(rot) - 3) if ps[m] == 2]
    for m in one:
        (ref, scale), d = _debug_record(eng, sets[so[2]:so[3]], rot[m], pos[m])
        assert int(rec[m, abi.SCORE_COUNT]) == int(d["ok"].sum())
        assert sk.record_err(rec[m], ref, scale) <= DEBUG_TOL


# ---- nothing else moves ----------------------------------------------------------------------------------------------
def test_map_and_staged_batch_untouched():
    cfg, blob, scans = scenes.box_scene("leg_fusion", batch=2)
    eng = Engine(cfg)
    eng.map_upload(blob)
    n0, n1 = len(scans[0]), len(scans[1])
    x = abi.default_states(2); P = abi.init_cov(2); Q = abi.process_cov_Q(cfg)
    args = (x, P, Q, np.zeros(2, abi.CLOCK_DTYPE), np.concatenate(scans), [0, n0, n0 + n1], [0.0, 0.0])
    eng.stage(*args)
    eng.run(iters=2)
    ref = eng.fetch()
    eng.stage(*args)
    before = eng.map_download()
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 940)
    _score(eng, scans[0], rot, pos)
    eng.run(iters=2)
    out = eng.fetch()
    for k in ("x", "P", "clk", "world", "n_eff"):
        assert np.asarray(out[k]).tobytes() == np.asarray(ref[k]).tobytes(), k
    _same_map(eng.map_download(), before)


def _same_map(a, b):
    """Byte-equal maps: header, nodes, aux and points as downloaded, the roots in key order (a download lists them in the
    order its threads claim them)."""
    pa, pb = abi.parse_map_blob(a), abi.parse_map_blob(b)
    assert pa[0].tobytes() == pb[0].tobytes()
    ra, rb = (np.sort(r.view(np.uint8).reshape(-1, 16).view("V16").ravel()) for r in (pa[1], pb[1]))
    assert ra.tobytes() == rb.tobytes()
    for k in (2, 3, 4):
        assert pa[k].tobytes() == pb[k].tobytes(), k


# ---- errors ----------------------------------------------------------------------------------------------------------
def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_errors_write_nothing():
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    pts = np.ascontiguousarray(scans[0][:600])
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 950)
    n = len(rot)
    so = np.array([0, 300, 600], np.uint32)
    ps = (np.arange(n) % 2).astype(np.uint32)
    rc, pc = np.ascontiguousarray(sk.ROT_COV), np.ascontiguousarray(sk.POS_COV)
    rot = np.ascontiguousarray(rot.reshape(n, 9)); pos = np.ascontiguousarray(pos)

    def call(eng, n_sets=2, pts=pts, so=so, n_poses=n, ps=ps, rot=rot, pos=pos, rc=rc, pc=pc):
        out = np.full((max(n_poses, 1), 32), 7.0)
        code = lib().lk_score_poses(eng.h, n_sets, _p(pts), _p(so), n_poses, _p(ps), _p(rot), _p(pos), _p(rc), _p(pc), _p(out))
        return code, bool((out == 7.0).all())

    fresh = Engine(cfg)
    assert call(fresh) == (-7, True)  # LK_ERR_NOT_READY: no map
    eng = Engine(cfg)
    eng.map_upload(blob)
    bad = lambda a, i, v: (lambda b: (b.reshape(-1).__setitem__(i, v), b)[1])(a.copy())  # noqa: E731
    cases = dict(pts=dict(pts=None), offsets=dict(so=None), pose_set=dict(ps=None), rot=dict(rot=None), pos=dict(pos=None),
                 rot_cov=dict(rc=None), pos_cov=dict(pc=None),
                 monotone=dict(so=np.array([0, 400, 300], np.uint32)), set_range=dict(ps=bad(ps, 3, 2)),
                 rot_nan=dict(rot=bad(rot, 5, np.nan)), pos_inf=dict(pos=bad(pos, 2, np.inf)), rot_cov_nan=dict(rc=bad(rc, 1, np.nan)),
                 pos_cov_inf=dict(pc=bad(pc, 8, -np.inf)))
    for what, kw in cases.items():
        assert call(eng, **kw) == (-1, True), what  # LK_ERR_INVALID_ARG
    # NULL sums_out
    assert lib().lk_score_poses(eng.h, 2, _p(pts), _p(so), n, _p(ps), _p(rot), _p(pos), _p(rc), _p(pc), None) == -1
    # n_poses == 0: nothing to do, even with NULL arguments, and nothing written
    assert call(eng, n_poses=0, pts=None, ps=None, rot=None) == (0, True)
    assert call(fresh, n_poses=0) == (0, True)
    # the handle stays usable
    code, untouched = call(eng)
    assert code == 0 and not untouched


# ---- the recipe of INTEGRATION.md §5 ---------------------------------------------------------------------------------
def test_recipe_recovers_the_pose():
    """A VLP-16 scan of the box room (square, so the yaw search stays within +-30 deg of the guess), taken 1.6 m and 20 deg
    from a rough guess: grid, score, top k by count, k one-bucket scans refined by lk_batch_run, re-score, best count."""
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw, pb)
    eng = Engine(cfg)
    eng.map_upload(o.map_export())
    true_rv, true_p = np.array([0.01, -0.015, 0.35]), np.array([1.1, -1.2, 0.03])
    pts = sc.scan(rotvec=true_rv, trans=true_p, ext_R=R, ext_t=t, blind=cfg["blind"], stream=960, **synth.VLP16)
    R_true = synth.exp_so3(true_rv)
    R_guess, p_guess = np.eye(3), np.zeros(3)  # 20 deg, 1.6 m off
    # 1-2. a grid around the guess, scored with a wide prior (the gate then admits points a grid step away)
    wide_rot, wide_pos = (np.deg2rad(2.0) ** 2) * np.eye(3), 0.1 ** 2 * np.eye(3)
    g = np.arange(-2.0, 2.01, 0.2)
    off = np.stack(np.meshgrid(g, g, [0.0], indexing="ij"), -1).reshape(-1, 3)
    rot, pos = sk.grid_poses(R_guess, p_guess, np.deg2rad(np.arange(-30.0, 30.1, 2.0)), off)
    rec = _score(eng, pts, rot, pos, rot_cov=wide_rot, pos_cov=wide_pos)
    # 3. top k by count
    k = 8
    top = np.argsort(-rec[:, abi.SCORE_COUNT], kind="stable")[:k]
    # 4. one-bucket scans at those poses, refined
    x = np.concatenate([sk.pose_state(rot[i], pos[i]) for i in top])
    P = np.tile(sk.pose_cov(wide_rot, wide_pos), (k, 1))
    n = len(pts)
    eng.stage(x, P, abi.process_cov_Q(cfg), np.zeros(k, abi.CLOCK_DTYPE), np.tile(pts, (k, 1)), np.arange(k + 1) * n, np.zeros(k))
    eng.run(iters=10)
    xr = eng.fetch(want_world=False)["x"]
    # 5. re-score the refined poses with the tight prior, keep the best
    rr = np.array([xr["rot"][i].reshape(3, 3) for i in range(k)]); pr = np.array([xr["pos"][i] for i in range(k)])
    rec2 = _score(eng, pts, rr, pr)
    b = int(np.argmax(rec2[:, abi.SCORE_COUNT]))
    d_pos = float(np.linalg.norm(pr[b] - true_p))
    d_rot = float(np.degrees(np.linalg.norm(lko.log_so3(R_true.T @ rr[b]))))
    mean_nr = rec2[b, abi.SCORE_SUM_Z2R] / rec2[b, abi.SCORE_COUNT]
    print(f"[score] recipe: {len(rot)} poses, best count {rec2[b, abi.SCORE_COUNT]:.0f} of {n}, position error {d_pos:.4f} m, "
          f"attitude error {d_rot:.4f} deg, mean normalised residual {mean_nr:.3f}")
    assert d_pos < 0.03 and d_rot < 0.3
    assert rec2[b, abi.SCORE_COUNT] > 0.8 * n
