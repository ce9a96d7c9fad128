"""lk_refine_poses on the device: its poses against the reference's chains (tests/golden/ref_refine_poses.npz), one step
against the numpy restatement on lk_score_poses' record, iters steps against the staged-copies composition it replaces
(lk_batch_stage + lk_batch_run(iters)); records bitwise lk_score_poses at the refined poses; bitwise invariance to the
other poses of the call; nothing else on the handle moves; the errors; and the localisation recipe of INTEGRATION.md §5
end to end, with the top 8 and with 256 starts."""
import ctypes as C

import numpy as np

import pytest

import lko
import refine_cases as rk
import score_cases as sk
import scenes
from legkilo_b200 import Engine, abi, lib, synth

pytestmark = pytest.mark.gpu
# Device pose against the reference's pose after the same number of steps (m / rad, largest entry of R and p): 100x the
# worst measured on an H100 80GB HBM3 (700 W), 2.2e-16
FIXTURE_TOL = 2.2e-14
# One device step against the numpy step on the same record: |difference| <= STEP_REL |delta| + STEP_ABS; worst measured
# on the H100: 9.3e-15 |delta|
STEP_REL, STEP_ABS = 1e-12, 1e-15
# Device pose against lk_batch_run(10) on the one-bucket scan at that pose (the sums differ in their order of addition):
# 100x the worst measured on the H100, 2.2e-16
COMPOSITION_TOL = 2.2e-14
WIDE_ROT, WIDE_POS = (np.deg2rad(2.0) ** 2) * np.eye(3), 0.1 ** 2 * np.eye(3)


def _refine(eng, pts, rot, pos, iters, set_offsets=None, pose_set=None, rot_cov=sk.ROT_COV, pos_cov=sk.POS_COV,
            want_records=True):
    so = [0, len(pts)] if set_offsets is None else set_offsets
    ps = np.zeros(len(rot), np.uint32) if pose_set is None else pose_set
    return eng.refine_poses(pts, so, ps, rot, pos, rot_cov, pos_cov, iters, want_records)


def _score(eng, pts, rot, pos, set_offsets=None, pose_set=None, rot_cov=sk.ROT_COV, pos_cov=sk.POS_COV):
    so = [0, len(pts)] if set_offsets is None else set_offsets
    ps = np.zeros(len(rot), np.uint32) if pose_set is None else pose_set
    return eng.score_poses(pts, so, ps, rot, pos, rot_cov, pos_cov)


def _near_poses(R0, p0, stream):
    g = synth.rng(stream)
    rots, poss = [R0], [np.asarray(p0, float)]
    for rs, ts in ((0.003, 0.01), (0.01, 0.05), (0.02, 0.1), (0.03, 0.2)):
        rots.append(synth.exp_so3(g.normal(0.0, rs, 3)) @ R0)
        poss.append(np.asarray(p0, float) + g.normal(0.0, ts, 3))
    return np.array(rots), np.array(poss)


def _box(batch=1):
    cfg, blob, scans = scenes.box_scene("leg_fusion", batch=batch)
    eng = Engine(cfg)
    eng.map_upload(blob)
    return eng, cfg, scans


def _composition(eng, cfg, sets, rot, pos, rot_cov, pos_cov, iters):
    """lk_batch_run(iters) on one-bucket scans of sets[m] staged at (rot[m], pos[m]), P from the symmetrised blocks."""
    M = len(rot)
    x = np.concatenate([sk.pose_state(rot[i], pos[i]) for i in range(M)])
    P = np.tile(sk.pose_cov(0.5 * (rot_cov + rot_cov.T), 0.5 * (pos_cov + pos_cov.T)), (M, 1))
    so = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.uint32)
    eng.stage(x, P, abi.process_cov_Q(cfg), np.zeros(M, abi.CLOCK_DTYPE), np.concatenate(sets), so, np.zeros(M))
    eng.run(iters=iters)
    xr = eng.fetch(want_world=False)["x"]
    return np.array([xr["rot"][i].reshape(3, 3) for i in range(M)]), np.array([xr["pos"][i] for i in range(M)])


def _pose_err(Ra, pa, Rb, pb):
    return float(max(np.abs(np.asarray(Ra) - Rb).max(), np.abs(np.asarray(pa) - pb).max()))


# ---- the reference's chains ------------------------------------------------------------------------------------------
def test_fixture_chains_equal_reference():
    d, g = sk.load_fixture(), rk.load_fixture()
    eng = Engine(abi.CONFIGS["leg_fusion"])
    eng.map_upload(d["blob"])
    rot0, pos0 = d["rot"][rk.POSES], d["pos"][rk.POSES]
    worst = 0.0
    for iters in range(1, rk.K + 1):
        rot, pos, rec = _refine(eng, d["pts"], rot0, pos0, iters, rot_cov=d["rot_cov"], pos_cov=d["pos_cov"])
        worst = max(worst, _pose_err(rot, pos, g["rot"][:, iters], g["pos"][:, iters]))
        if iters < rk.K:  # the record at the refined pose is the reference's next call's count
            np.testing.assert_array_equal(rec[:, abi.SCORE_COUNT].astype(np.int64), g["counts"][:, iters])
    print(f"[refine] fixture: worst pose error against the reference's chains {worst:.3g}")
    assert worst <= FIXTURE_TOL


# ---- one step against the host restatement ---------------------------------------------------------------------------
def test_one_step_equals_host_restatement():
    eng, cfg, scans = _box()
    pts = scans[0]
    # single points as sets of their own: the first that scores one row at the identity is the count-1 case
    singles = pts[:200]
    rec1 = _score(eng, singles, np.tile(np.eye(3), (200, 1, 1)), np.zeros((200, 3)), np.arange(201), np.arange(200))
    one = int(np.flatnonzero(rec1[:, abi.SCORE_COUNT] == 1)[0])
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 970)
    rot = np.concatenate([rot, rot[:1], rot[1:2]]); pos = np.concatenate([pos, pos[:1], pos[1:2] + 1000.0])  # +1: off the map
    sets = np.concatenate([pts, pts[one:one + 1]])
    so = [0, len(pts), len(pts) + 1]
    ps = np.array([0] * (len(rot) - 2) + [1, 0], np.uint32)
    before = _score(eng, sets, rot, pos, so, ps)
    assert before[-2, abi.SCORE_COUNT] == 1 and before[-1, abi.SCORE_COUNT] == 0
    ro, po, _ = _refine(eng, sets, rot, pos, 1, so, ps)
    assert ro[-1].tobytes() == rot[-1].tobytes() and po[-1].tobytes() == pos[-1].tobytes()
    worst = 0.0
    for m in range(len(rot) - 1):
        delta = rk.step_delta(before[m], sk.ROT_COV, sk.POS_COV)
        Rh, ph = rk.boxplus(rot[m], pos[m], delta)
        err = _pose_err(ro[m], po[m], Rh, ph)
        worst = max(worst, err / np.abs(delta).max())
        assert err <= STEP_REL * np.abs(delta).max() + STEP_ABS, (m, err, np.abs(delta).max())
    print(f"[refine] one step against the host restatement: worst error / |delta| {worst:.3g}")


# ---- against the staged-copies composition ---------------------------------------------------------------------------
def _recipe_scene():
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
    g = np.arange(-2.0, 2.01, 0.2)
    off = np.stack(np.meshgrid(g, g, [0.0], indexing="ij"), -1).reshape(-1, 3)
    rot, pos = sk.grid_poses(np.eye(3), np.zeros(3), np.deg2rad(np.arange(-30.0, 30.1, 2.0)), off)
    return eng, cfg, pts, synth.exp_so3(true_rv), true_p, rot, pos


def test_recipe_top8_equals_composition():
    eng, cfg, pts, _, _, rot, pos = _recipe_scene()
    rec = _score(eng, pts, rot, pos, rot_cov=WIDE_ROT, pos_cov=WIDE_POS)
    top = np.argsort(-rec[:, abi.SCORE_COUNT], kind="stable")[:8]
    ro, po, _ = _refine(eng, pts, rot[top], pos[top], 10, rot_cov=WIDE_ROT, pos_cov=WIDE_POS, want_records=False)
    rc, pc = _composition(eng, cfg, [pts] * 8, rot[top], pos[top], WIDE_ROT, WIDE_POS, 10)
    err = _pose_err(ro, po, rc, pc)
    print(f"[refine] recipe top 8 against lk_batch_run(10): {err:.3g}")
    assert err <= COMPOSITION_TOL


def test_ragged_sets_equal_composition():
    eng, cfg, scans = _box()
    pts = scans[0]
    sizes = [300, 0, 1, 2000, 255, 257, 5000]
    so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    sets = pts[::3][:sum(sizes)]
    assert len(sets) == sum(sizes)
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 980)
    rot = np.concatenate([rot] * 3); pos = np.concatenate([pos] * 3)
    ps = (np.arange(len(rot)) % 7).astype(np.uint32)
    # asymmetric blocks: the call and the composition both use their symmetric parts
    rc_in, pc_in = sk.ROT_COV + np.triu(sk.ROT_COV, 1) * 0.1, sk.POS_COV + np.tril(sk.POS_COV, -1) * 0.1
    ro, po, rec = _refine(eng, sets, rot, pos, 10, so, ps, rc_in, pc_in)
    empty = ps == 1
    assert ro[empty].tobytes() == rot[empty].tobytes() and po[empty].tobytes() == pos[empty].tobytes()
    assert (rec[empty] == 0).all()
    keep = np.flatnonzero(~empty)
    rcmp, pcmp = _composition(eng, cfg, [sets[so[ps[m]]:so[ps[m] + 1]] for m in keep], rot[keep], pos[keep], rc_in, pc_in, 10)
    err = _pose_err(ro[keep], po[keep], rcmp, pcmp)
    print(f"[refine] ragged sets against lk_batch_run(10): {err:.3g}")
    assert err <= COMPOSITION_TOL
    for m in keep:  # each pose refined alone: bitwise
        s = int(ps[m])
        a = _refine(eng, sets[so[s]:so[s + 1]], rot[m:m + 1], pos[m:m + 1], 10, rot_cov=rc_in, pos_cov=pc_in)
        assert a[0].tobytes() == ro[m:m + 1].tobytes() and a[1].tobytes() == po[m:m + 1].tobytes()
        assert a[2].tobytes() == rec[m:m + 1].tobytes(), m


# ---- bitwise properties ----------------------------------------------------------------------------------------------
def test_records_are_score_at_refined_poses():
    eng, cfg, scans = _box()
    pts = scans[0]
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 990)
    ro, po, rec = _refine(eng, pts, rot, pos, 4)
    assert rec.tobytes() == _score(eng, pts, ro, po).tobytes()
    ro2, po2, none = _refine(eng, pts, rot, pos, 4, want_records=False)
    assert none is None and ro2.tobytes() == ro.tobytes() and po2.tobytes() == po.tobytes()
    # outputs aliasing the inputs
    so, ps = np.array([0, len(pts)], np.uint32), np.zeros(len(rot), np.uint32)
    r = np.ascontiguousarray(rot.reshape(-1, 9)).copy(); p = np.ascontiguousarray(pos).copy()
    rc, pc = np.ascontiguousarray(sk.ROT_COV), np.ascontiguousarray(sk.POS_COV)
    pts4 = np.ascontiguousarray(pts, np.float32)
    code = lib().lk_refine_poses(eng.h, 1, _p(pts4), _p(so), len(rot), _p(ps), _p(r), _p(p), _p(rc), _p(pc), 4, _p(r), _p(p),
                                 None)
    assert code == 0 and r.tobytes() == ro.reshape(-1, 9).tobytes() and p.tobytes() == po.tobytes()


def test_pose_does_not_depend_on_the_other_poses():
    """4 096 poses of one 28 800-point scan (two windows), against each pose refined alone, the call in reversed order, a
    second run and a mixed call: bitwise."""
    eng, cfg, scans = _box()
    pts = scans[0]
    assert len(pts) > 28000
    off = np.stack(np.meshgrid(np.linspace(-0.3, 0.3, 16), np.linspace(-0.3, 0.3, 16), [0.0], indexing="ij"), -1).reshape(-1, 3)
    rot, pos = sk.grid_poses(np.eye(3), np.zeros(3), np.linspace(-0.1, 0.1, 16), off)
    assert len(rot) == 4096
    ro, po, rec = _refine(eng, pts, rot, pos, 3)
    out = np.concatenate([ro.reshape(-1, 9), po, rec], 1)
    rr = _refine(eng, pts, rot[::-1], pos[::-1], 3)
    assert np.concatenate([rr[0].reshape(-1, 9), rr[1], rr[2]], 1)[::-1].tobytes() == out.tobytes()
    again = _refine(eng, pts, rot, pos, 3)
    assert np.concatenate([again[0].reshape(-1, 9), again[1], again[2]], 1).tobytes() == out.tobytes()
    rows_per_pose = (len(pts) + 255) // 256
    boundary = ((1 << 18) // (16 * rows_per_pose)) * 16  # first pose of the second window
    for i in (0, 1, 15, 16, boundary - 1, boundary, 4095):
        a = _refine(eng, pts, rot[i:i + 1], pos[i:i + 1], 3)
        assert np.concatenate([a[0].reshape(-1, 9), a[1], a[2]], 1).tobytes() == out[i:i + 1].tobytes(), i
    idx = np.array([4095, 7, boundary, 3, boundary - 1])
    so = [0, len(pts), 2 * len(pts)]
    mix = _refine(eng, np.concatenate([pts, pts[::-1]]), np.repeat(rot[idx], 2, 0), np.repeat(pos[idx], 2, 0), 3, so,
                  np.tile([0, 1], len(idx)).astype(np.uint32))
    assert np.concatenate([mix[0].reshape(-1, 9), mix[1], mix[2]], 1)[0::2].tobytes() == out[idx].tobytes()


def test_map_staged_batch_and_stats_untouched():
    eng, cfg, scans = _box(batch=2)
    n0, n1 = len(scans[0]), len(scans[1])
    x = abi.default_states(2); P = abi.init_cov(2); Q = abi.process_cov_Q(cfg)
    args = (x, P, Q, np.zeros(2, abi.CLOCK_DTYPE), np.concatenate(scans), [0, n0, n0 + n1], [0.0, 0.0])
    eng.stage(*args)
    eng.run(iters=2)
    ref = eng.fetch()
    eng.stage(*args)
    before, stats = eng.map_download(), eng.map_stats()
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 1000)
    _refine(eng, scans[0], rot, pos, 5)
    assert eng.map_stats() == stats
    eng.run(iters=2)
    out = eng.fetch()
    for k in ("x", "P", "clk", "world", "n_eff"):
        assert np.asarray(out[k]).tobytes() == np.asarray(ref[k]).tobytes(), k
    pa, pb = abi.parse_map_blob(eng.map_download()), abi.parse_map_blob(before)
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
    rot, pos = _near_poses(np.eye(3), np.zeros(3), 1010)
    n = len(rot)
    so = np.array([0, 300, 600], np.uint32)
    ps = (np.arange(n) % 2).astype(np.uint32)
    rc, pc = np.ascontiguousarray(sk.ROT_COV), np.ascontiguousarray(sk.POS_COV)
    rot = np.ascontiguousarray(rot.reshape(n, 9)); pos = np.ascontiguousarray(pos)

    def call(eng, n_sets=2, pts=pts, so=so, n_poses=n, ps=ps, rot=rot, pos=pos, rc=rc, pc=pc, iters=3, ro=True, po=True):
        k = max(n_poses, 1)
        r_out, p_out, s_out = np.full((k, 9), 7.0), np.full((k, 3), 7.0), np.full((k, 32), 7.0)
        code = lib().lk_refine_poses(eng.h, n_sets, _p(pts), _p(so), n_poses, _p(ps), _p(rot), _p(pos), _p(rc), _p(pc),
                                     iters, _p(r_out) if ro else None, _p(p_out) if po else None, _p(s_out))
        return code, bool((r_out == 7.0).all() and (p_out == 7.0).all() and (s_out == 7.0).all())

    fresh = Engine(cfg)
    assert call(fresh) == (-7, True)  # LK_ERR_NOT_READY: no map
    eng = Engine(cfg)
    eng.map_upload(blob)
    bad = lambda a, i, v: (lambda b: (b.reshape(-1).__setitem__(i, v), b)[1])(a.copy())  # noqa: E731
    cases = dict(pts=dict(pts=None), offsets=dict(so=None), pose_set=dict(ps=None), rot=dict(rot=None), pos=dict(pos=None),
                 rot_cov=dict(rc=None), pos_cov=dict(pc=None), rot_out=dict(ro=False), pos_out=dict(po=False),
                 monotone=dict(so=np.array([0, 400, 300], np.uint32)), set_range=dict(ps=bad(ps, 3, 2)),
                 rot_nan=dict(rot=bad(rot, 5, np.nan)), pos_inf=dict(pos=bad(pos, 2, np.inf)), rot_cov_nan=dict(rc=bad(rc, 1, np.nan)),
                 pos_cov_inf=dict(pc=bad(pc, 8, -np.inf)), iters_0=dict(iters=0), iters_neg=dict(iters=-2))
    for what, kw in cases.items():
        assert call(eng, **kw) == (-1, True), what  # LK_ERR_INVALID_ARG
    # n_poses == 0: nothing to do, even with NULL arguments, and nothing written
    assert call(eng, n_poses=0, pts=None, ps=None, rot=None) == (0, True)
    assert call(fresh, n_poses=0) == (0, True)
    # the handle stays usable
    code, untouched = call(eng)
    assert code == 0 and not untouched


# ---- the recipe of INTEGRATION.md §5 ---------------------------------------------------------------------------------
def _best(eng, pts, rr, pr, R_true, true_p):
    rec = _score(eng, pts, rr, pr)
    b = int(np.argmax(rec[:, abi.SCORE_COUNT]))
    d_pos = float(np.linalg.norm(pr[b] - true_p))
    d_rot = float(np.degrees(np.linalg.norm(lko.log_so3(R_true.T @ rr[b]))))
    return b, rec, d_pos, d_rot


def test_recipe_recovers_the_pose():
    """The scan of test_gpu_score_poses.test_recipe_recovers_the_pose (1.6 m and 20 deg off the guess): score the grid
    wide, refine the top 8 wide with iters = 10, re-score them tight, keep the best. No staged batch."""
    eng, cfg, pts, R_true, true_p, rot, pos = _recipe_scene()
    assert len(rot) == 13671
    rec = _score(eng, pts, rot, pos, rot_cov=WIDE_ROT, pos_cov=WIDE_POS)
    top = np.argsort(-rec[:, abi.SCORE_COUNT], kind="stable")[:8]
    rr, pr, _ = _refine(eng, pts, rot[top], pos[top], 10, rot_cov=WIDE_ROT, pos_cov=WIDE_POS, want_records=False)
    b, rec2, d_pos, d_rot = _best(eng, pts, rr, pr, R_true, true_p)
    print(f"[refine] recipe: best count {rec2[b, abi.SCORE_COUNT]:.0f} of {len(pts)}, position error {d_pos:.4f} m, "
          f"attitude error {d_rot:.4f} deg")
    assert d_pos < 0.03 and d_rot < 0.3
    assert rec2[b, abi.SCORE_COUNT] > 0.8 * len(pts)


def test_multi_start_recovers_the_pose():
    eng, cfg, pts, R_true, true_p, rot, pos = _recipe_scene()
    rec = _score(eng, pts, rot, pos, rot_cov=WIDE_ROT, pos_cov=WIDE_POS)
    top = np.argsort(-rec[:, abi.SCORE_COUNT], kind="stable")[:256]
    rr, pr, _ = _refine(eng, pts, rot[top], pos[top], 10, rot_cov=WIDE_ROT, pos_cov=WIDE_POS, want_records=False)
    b, rec2, d_pos, d_rot = _best(eng, pts, rr, pr, R_true, true_p)
    near = int(sum(np.linalg.norm(pr[i] - true_p) < 0.03 for i in range(len(top))))
    print(f"[refine] multi-start: 256 starts, {near} within 0.03 m; best position error {d_pos:.4f} m, attitude error "
          f"{d_rot:.4f} deg")
    assert d_pos < 0.03 and d_rot < 0.3
