"""lk_search_poses on the device: bitwise the composition it replaces (tests/search_cases.py: the numpy lattice through
lk_score_poses wide, the best k per set, lk_refine_poses, lk_score_poses tight, the stable order by tight count) on the
recipe scene, on ragged calls, on ties and over 2^24 candidates; each set's outputs independent of the other sets; the
scorer's scratch independent of the number of candidates; nothing else on the handle moves; the errors; and the recipe of
INTEGRATION.md §5 end to end on one and on 16 scans."""
import ctypes as C

import numpy as np

import pytest

import lko
import search_cases as xs
import scenes
from legkilo_b200 import Engine, abi, lib, synth

pytestmark = pytest.mark.gpu

RECIPE_ATT = xs.yaw_attitudes(np.arange(-30.0, 30.1, 2.0))  # 31 attitudes
RECIPE_STEP, RECIPE_COUNTS = np.array([0.2, 0.2, 1.0]), np.array([21, 21, 1], np.uint32)
RECIPE_ORIGIN = np.array([-2.0, -2.0, 0.0])


def _recipe_scene(true_rv=(0.01, -0.015, 0.35), true_p=(1.1, -1.2, 0.03), stream=960, eng=None):
    """The box room and VLP-16 scan of test_gpu_refine_poses._recipe_scene (1.6 m and 20 deg off the guess)."""
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    if eng is None:
        pw, pb = sc.map_points(ext_R=R, ext_t=t)
        o = lko.Oracle(cfg)
        o.build_voxel_map(pw, pb)
        eng = Engine(cfg)
        eng.map_upload(o.map_export())
    pts = sc.scan(rotvec=np.asarray(true_rv), trans=np.asarray(true_p), ext_R=R, ext_t=t, blind=cfg["blind"], stream=stream,
                  **synth.VLP16)
    return eng, np.ascontiguousarray(pts, np.float32), synth.exp_so3(np.asarray(true_rv)), np.asarray(true_p)


def _search(eng, pts, so, ao, att, origin, step, counts, iters, k):
    return eng.search_poses(pts, so, ao, att, origin, step, counts, xs.WIDE_ROT, xs.WIDE_POS, iters, xs.TIGHT_ROT,
                            xs.TIGHT_POS, k)


def _both(eng, pts, so, ao, att, origin, step, counts, iters, k, **kw):
    out = _search(eng, pts, so, ao, att, origin, step, counts, iters, k)
    ref = xs.compose(eng, pts, so, ao, att, origin, step, counts, iters, k, **kw)
    return out, ref


# ---- bitwise against the composition ---------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [8, 256])
def test_recipe_equals_composition(k):
    eng, pts, _, _ = _recipe_scene()
    out, ref = _both(eng, pts, [0, len(pts)], [0, 31], RECIPE_ATT, RECIPE_ORIGIN[None], RECIPE_STEP, RECIPE_COUNTS, 10, k)
    assert xs.same(out, ref)
    assert len(np.unique(out[3])) == k


def _ragged():
    """Sets of 2 000, 0, 1, 300 points, a 28 734-point scan with 2 400 candidates (two windows: 271 200 partial rows), and
    40 sets of 300 points with 4 attitudes each (one window holds them all); 2 x 2 x 1 lattice, k = 8."""
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    eng = Engine(cfg)
    eng.map_upload(blob)
    scan = np.ascontiguousarray(scans[0], np.float32)
    g = synth.rng(1200)
    sizes = [2000, 0, 1, 300, len(scan)] + [300] * 40
    n_att = [5, 3, 5, 2, 600] + [4] * 40  # set 3: exactly k = 8 candidates
    sets = [scan[:2000], scan[:0], scan[100:101], scan[::7][:300], scan] + [scan[i * 300:(i + 1) * 300] for i in range(40)]
    pts = np.concatenate(sets)
    so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    ao = np.concatenate([[0], np.cumsum(n_att)]).astype(np.uint32)
    att = np.array([synth.exp_so3(g.normal(0.0, 0.05, 3)) for _ in range(int(ao[-1]))])
    origin = g.normal(0.0, 0.1, (len(sizes), 3))
    return eng, pts, so, ao, att, origin, np.array([0.05, 0.07, 0.0]), np.array([2, 2, 1], np.uint32)


def test_ragged_sets_equal_composition():
    eng, pts, so, ao, att, origin, step, counts = _ragged()
    out, ref = _both(eng, pts, so, ao, att, origin, step, counts, 3, 8)
    assert xs.same(out, ref)
    assert (out[2][1] == 0).all() and (out[3][1] == np.arange(8)).all()  # the empty set: every count 0, kept by index
    assert sorted(out[3][3]) == list(range(8))  # exactly k candidates: all kept


def test_each_set_alone_and_permuted():
    eng, pts, so, ao, att, origin, step, counts = _ragged()
    out = _search(eng, pts, so, ao, att, origin, step, counts, 3, 8)
    n = len(so) - 1
    perm = synth.rng(1210).permutation(n)
    sets = [pts[so[s]:so[s + 1]] for s in perm]
    atts = [att[ao[s]:ao[s + 1]] for s in perm]
    pso = np.concatenate([[0], np.cumsum([len(x) for x in sets])]).astype(np.uint32)
    pao = np.concatenate([[0], np.cumsum([len(x) for x in atts])]).astype(np.uint32)
    p = _search(eng, np.concatenate(sets), pso, pao, np.concatenate(atts), origin[perm], step, counts, 3, 8)
    for j, s in enumerate(perm):
        assert all(p[i][j].tobytes() == out[i][s].tobytes() for i in range(4)), s
    for s in (0, 1, 2, 3, 4, 20):
        a = _search(eng, pts[so[s]:so[s + 1]], [0, so[s + 1] - so[s]], [0, ao[s + 1] - ao[s]], att[ao[s]:ao[s + 1]],
                    origin[s:s + 1], step, counts, 3, 8)
        assert all(a[i][0].tobytes() == out[i][s].tobytes() for i in range(4)), s


def test_ties_follow_the_candidate_index():
    eng, pts, _, _ = _recipe_scene()
    # far from the map: every count 0, the keep is candidates 0 .. k-1
    out, ref = _both(eng, pts, [0, len(pts)], [0, 3], RECIPE_ATT[:3], np.array([[500.0, 500.0, 0.0]]), RECIPE_STEP,
                     RECIPE_COUNTS, 2, 16)
    assert xs.same(out, ref) and (out[3][0] == np.arange(16)).all() and (out[2] == 0).all()
    # one attitude repeated and a lattice of step 0: every candidate the same pose, one positive count for all
    att = np.repeat(RECIPE_ATT[15:16], 6, 0)
    out, ref = _both(eng, pts, [0, len(pts)], [0, 6], att, np.array([[1.0, -1.0, 0.0]]), np.zeros(3),
                     np.array([3, 2, 1], np.uint32), 2, 20)
    assert xs.same(out, ref)
    assert out[2][0, 0, abi.SCORE_COUNT] > 0 and (out[3][0] == np.arange(20)).all()


# ---- memory that does not grow with the candidates ---------------------------------------------------------------------
def test_scratch_does_not_depend_on_the_candidates():
    """Two sets of 1 024 points (4 chunks each): 2^16 candidates fill one window, 2^24 take 256; the scorer's scratch is
    the same after both and within the header's bound, and the 2^24 search equals the composition over slices of 2^20."""
    eng, pts, R_true, true_p = _recipe_scene()
    sets = np.ascontiguousarray(np.concatenate([pts[:1024], pts[5000:6024]]))
    so, ao = np.array([0, 1024, 2048], np.uint32), np.array([0, 1, 2], np.uint32)
    att = np.array([R_true, RECIPE_ATT[16]])
    origin = np.array([true_p - [0.64, 1.28, 1.28], [-0.5, -0.5, -0.5]])
    step = np.array([0.01, 0.01, 0.01])
    k = 32
    small = _search(eng, sets, so, ao, att, origin, step, np.array([32, 32, 32], np.uint32), 4, k)
    held = eng.scorer_scratch()
    big = _search(eng, sets, so, ao, att, origin, step, np.array([128, 256, 256], np.uint32), 4, k)
    assert eng.scorer_scratch() == held
    # the header's bound: 16 B per point, 72 B per set and attitude, 1 024 B per kept pose + 32 B per (chunk, tile) of
    # them, 192 MiB for a window, each buffer with 1/8 slack and 256 B
    n_keep = 2 * k
    bound = 16 * 2048 + 72 * 4 + 1024 * n_keep + 32 * 2 * 4 * ((k + 15) // 16) + (192 << 20)
    print(f"[search] scorer scratch: {held[0] / 2**20:.1f} MiB device, {held[1] / 2**10:.1f} KiB page-locked; "
          f"bound {bound * 9 / 8 / 2**20:.1f} MiB")
    assert held[0] <= bound * 9 // 8 + 16 * 256
    assert held[1] <= (72 * 4 + 16 * n_keep + 32 * 2 * 4 * 2 + 356 * n_keep + 4 * 256) * 5 // 4 + 4096
    ref = xs.compose(eng, sets, so, ao, att, origin, step, np.array([128, 256, 256], np.uint32), 4, k, slice_=1 << 20)
    assert xs.same(big, ref)
    assert small[3].max() < 1 << 15 and big[3].max() < 1 << 23


# ---- end to end --------------------------------------------------------------------------------------------------------
def test_recipe_recovers_the_pose():
    eng, pts, R_true, true_p = _recipe_scene()
    rot, pos, rec, _ = _search(eng, pts, [0, len(pts)], [0, 31], RECIPE_ATT, RECIPE_ORIGIN[None], RECIPE_STEP,
                               RECIPE_COUNTS, 10, 8)
    d_pos = float(np.linalg.norm(pos[0, 0] - true_p))
    d_rot = float(np.degrees(np.linalg.norm(lko.log_so3(R_true.T @ rot[0, 0]))))
    print(f"[search] recipe: best tight count {rec[0, 0, abi.SCORE_COUNT]:.0f} of {len(pts)}, position error {d_pos:.4f} m, "
          f"attitude error {d_rot:.4f} deg")
    assert d_pos < 0.03 and d_rot < 0.3
    assert rec[0, 0, abi.SCORE_COUNT] > 0.8 * len(pts)


def test_sixteen_scans_in_one_call():
    g = synth.rng(1220)
    eng, truths, scans = None, [], []
    for i in range(16):
        rv = np.array([g.normal(0.0, 0.01), g.normal(0.0, 0.01), np.deg2rad(g.uniform(-25.0, 25.0))])
        p = np.array([g.uniform(-1.5, 1.5), g.uniform(-1.5, 1.5), 0.03])
        eng, pts, R, t = _recipe_scene(rv, p, 1300 + i, eng)
        truths.append((R, t))
        scans.append(pts)
    so = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    ao = (np.arange(17) * 31).astype(np.uint32)
    rot, pos, rec, _ = _search(eng, np.concatenate(scans), so, ao, np.tile(RECIPE_ATT, (16, 1, 1)),
                               np.tile(RECIPE_ORIGIN, (16, 1)), RECIPE_STEP, RECIPE_COUNTS, 10, 8)
    for s, (R, t) in enumerate(truths):
        d_pos = float(np.linalg.norm(pos[s, 0] - t))
        d_rot = float(np.degrees(np.linalg.norm(lko.log_so3(R.T @ rot[s, 0]))))
        print(f"[search] scan {s}: position error {d_pos:.4f} m, attitude error {d_rot:.4f} deg")
        assert d_pos < 0.03 and d_rot < 0.3, s
        assert rec[s, 0, abi.SCORE_COUNT] > 0.8 * len(scans[s]), s


# ---- nothing else moves ------------------------------------------------------------------------------------------------
def test_map_staged_batch_and_stats_untouched():
    cfg, blob, scans = scenes.box_scene("leg_fusion", batch=2)
    eng = Engine(cfg)
    eng.map_upload(blob)
    n0, n1 = len(scans[0]), len(scans[1])
    x = abi.default_states(2); P = abi.init_cov(2); Q = abi.process_cov_Q(cfg)
    args = (x, P, Q, np.zeros(2, abi.CLOCK_DTYPE), np.concatenate(scans), [0, n0, n0 + n1], [0.0, 0.0])
    eng.stage(*args)
    eng.run(iters=2)
    ref = eng.fetch()
    rot, pos = RECIPE_ATT[[10, 15, 20]], np.array([[0.0, 0.0, 0.0], [0.1, 0.0, 0.0], [0.0, -0.1, 0.0]])
    score_before = eng.score_poses(scans[0], [0, n0], np.zeros(3, np.uint32), rot, pos, xs.WIDE_ROT, xs.WIDE_POS)
    eng.stage(*args)
    before, stats = eng.map_download(), eng.map_stats()
    _search(eng, scans[0], [0, n0], [0, 31], RECIPE_ATT, RECIPE_ORIGIN[None], RECIPE_STEP, RECIPE_COUNTS, 3, 8)
    assert eng.map_stats() == stats
    pa, pb = abi.parse_map_blob(eng.map_download()), abi.parse_map_blob(before)
    assert pa[0].tobytes() == pb[0].tobytes()
    ra, rb = (np.sort(r.view(np.uint8).reshape(-1, 16).view("V16").ravel()) for r in (pa[1], pb[1]))
    assert ra.tobytes() == rb.tobytes()
    for i in (2, 3, 4):
        assert pa[i].tobytes() == pb[i].tobytes(), i
    eng.run(iters=2)
    out = eng.fetch()
    for key in ("x", "P", "clk", "world", "n_eff"):
        assert np.asarray(out[key]).tobytes() == np.asarray(ref[key]).tobytes(), key
    # the scorer's shared scratch: a following lk_score_poses is still bitwise
    after = eng.score_poses(scans[0], [0, n0], np.zeros(3, np.uint32), rot, pos, xs.WIDE_ROT, xs.WIDE_POS)
    assert after.tobytes() == score_before.tobytes()


# ---- errors ------------------------------------------------------------------------------------------------------------
def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_errors_write_nothing():
    cfg, blob, scans = scenes.box_scene("leg_fusion")
    pts = np.ascontiguousarray(scans[0][:600], np.float32)
    so, ao = np.array([0, 300, 600], np.uint32), np.array([0, 2, 5], np.uint32)
    att = np.ascontiguousarray(RECIPE_ATT[:5].reshape(5, 9))
    origin = np.zeros((2, 3))
    step, counts = np.array([0.1, 0.1, 0.1]), np.array([2, 2, 1], np.uint32)
    wr, wp = np.ascontiguousarray(xs.WIDE_ROT), np.ascontiguousarray(xs.WIDE_POS)
    tr, tp = np.ascontiguousarray(xs.TIGHT_ROT), np.ascontiguousarray(xs.TIGHT_POS)

    def call(eng, n_sets=2, pts=pts, so=so, ao=ao, att=att, origin=origin, step=step, counts=counts, wr=wr, wp=wp, iters=2,
             tr=tr, tp=tp, k=4, outs=(True, True, True, True)):
        n = max(n_sets, 1) * 300
        bufs = [np.full((n, 9), 7.0), np.full((n, 3), 7.0), np.full((n, 32), 7.0), np.full(n, 7, np.uint32)]
        code = lib().lk_search_poses(eng.h, n_sets, _p(pts), _p(so), _p(ao), _p(att), _p(origin), _p(step), _p(counts),
                                     _p(wr), _p(wp), iters, _p(tr), _p(tp), k,
                                     *[_p(b) if o else None for b, o in zip(bufs, outs)])
        return code, all(bool((b == 7).all()) for b in bufs)

    fresh = Engine(cfg)
    assert call(fresh) == (-7, True)  # LK_ERR_NOT_READY: no map
    eng = Engine(cfg)
    eng.map_upload(blob)
    bad = lambda a, i, v: (lambda b: (b.reshape(-1).__setitem__(i, v), b)[1])(a.copy())  # noqa: E731
    cases = dict(pts=dict(pts=None), set_offsets=dict(so=None), att_offsets=dict(ao=None), att=dict(att=None),
                 origin=dict(origin=None), step=dict(step=None), counts=dict(counts=None), rot_cov=dict(wr=None),
                 pos_cov=dict(wp=None), rot_cov_tight=dict(tr=None), pos_cov_tight=dict(tp=None),
                 rot_out=dict(outs=(False, True, True, True)), pos_out=dict(outs=(True, False, True, True)),
                 sums_out=dict(outs=(True, True, False, True)), cand_out=dict(outs=(True, True, True, False)),
                 so_monotone=dict(so=np.array([0, 400, 300], np.uint32)), ao_monotone=dict(ao=np.array([0, 3, 2], np.uint32)),
                 counts_zero=dict(counts=bad(counts, 2, 0)), k_zero=dict(k=0), k_big=dict(k=257), iters_0=dict(iters=0),
                 iters_neg=dict(iters=-1), att_nan=dict(att=bad(att, 40, np.nan)), origin_inf=dict(origin=bad(origin, 4, np.inf)),
                 step_nan=dict(step=bad(step, 1, np.nan)), wr_nan=dict(wr=bad(wr, 3, np.nan)), wp_inf=dict(wp=bad(wp, 0, -np.inf)),
                 tr_nan=dict(tr=bad(tr, 8, np.nan)), tp_nan=dict(tp=bad(tp, 4, np.nan)),
                 fewer_than_k=dict(k=9),  # set 0: 2 attitudes x 4 = 8 candidates
                 too_many=dict(counts=np.array([1 << 16, 1 << 15, 1], np.uint32)))  # set 1: 3 x 2^31
    for what, kw in cases.items():
        assert call(eng, **kw) == (-1, True), what  # LK_ERR_INVALID_ARG
    # n_sets == 0: nothing to do, even with NULL arguments, and nothing written
    assert call(eng, n_sets=0, pts=None, so=None, att=None) == (0, True)
    assert call(fresh, n_sets=0) == (0, True)
    # the handle stays usable
    code, untouched = call(eng)
    assert code == 0 and not untouched
