"""lk_map_insert on the device: UpdateVoxelMap of point sets at known poses, many sets per call, cut into fixed-size
windows that each run through the slice-and-sort insert.

1. against the reference's fixtures (tests/golden/ref_map_insert.npz) and the CPU oracle;
2. replay of a streaming run: the poses and P blocks a streaming handle ended each bucket with, inserted in one call on a
   second handle, give the streaming map bitwise;
3. window boundaries: one call over several windows, one call per set, and sets split at arbitrary points across calls
   give the same map bitwise;
4. the hot plane images of inserted maps, through every kernel that reads them (tests/test_gpu_map_images.py: _probe);
5. storage: freezes and cuts recycle tiles, a slide between calls recycles the window, repeated insertion of a static
   scene stops growing the pools;
6. host behaviour: a staged batch survives the call, invalid arguments, n_sets = 0."""
import ctypes as C

import numpy as np
import pytest

import general_prior as gp
import lko_insert
import map_insert_cases as mic
import mapcmp
import scenes
import test_gpu_map_images as mi
import test_gpu_map_memory as mm
from legkilo_b200 import Engine, LkError, abi, lib, synth
from test_map_insert_oracle import fixture

pytestmark = pytest.mark.gpu
WINDOW = 32768  # lk_api.cu: MAP_INSERT_WINDOW


def exact(a, b):
    """Two map blobs equal in every field, matched by root key and octree path (node and point numbering may differ)."""
    _, ra, na, aa, pa = abi.parse_map_blob(a)
    _, rb, nb, ab, pb = abi.parse_map_blob(b)
    ka = {tuple(int(v) for v in r["key"]): int(r["node"]) for r in ra}
    kb = {tuple(int(v) for v in r["key"]): int(r["node"]) for r in rb}
    assert set(ka) == set(kb), (len(ka), len(kb))
    n = 0

    def walk(i, j, path):
        nonlocal n
        A, B, XA, XB = na[i:i + 1].copy(), nb[j:j + 1].copy(), aa[i:i + 1].copy(), ab[j:j + 1].copy()
        for R in (A, B):
            R["child_base"] = 0
            R["pad"] = 0
        for X in (XA, XB):
            X["pts_base"] = 0
            X["parent"] = 0
            X["pad"] = 0
        assert A.tobytes() == B.tobytes(), (path, A, B)
        assert XA.tobytes() == XB.tobytes(), (path, XA, XB)
        c, oa, ob = int(aa[i]["pts_count"]), int(aa[i]["pts_base"]), int(ab[j]["pts_base"])
        assert pa[oa:oa + c].tobytes() == pb[ob:ob + c].tobytes(), path
        n += 1
        f = int(na[i]["flags"])
        for k in range(8):
            if (f >> abi.NODE_CHILDMASK_SHIFT) & (1 << k):
                walk(int(na[i]["child_base"]) + k, int(nb[j]["child_base"]) + k, path + (k,))

    for key in sorted(ka):
        walk(ka[key], kb[key], (key,))
    return n


def _engine(cfg, blob=None):
    eng = Engine(cfg)
    if blob is not None:
        eng.map_upload(blob)
    return eng


# ---- 1. reference fixtures and oracle -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", mic.NAMES)
def test_device_matches_fixture_and_oracle(name):
    cfg, c, _, map1 = fixture(name)
    blob0 = mic.start_blob(cfg, c)
    eng = _engine(cfg, blob0)
    eng.map_insert(*mic.call(c))
    dev = eng.map_download()
    mapcmp.compare_digest(map1, dev)
    st = mapcmp.compare_blobs(mic.oracle_insert(cfg, blob0, *mic.call(c)), dev)
    assert st["planes"] > 100 and st["points"] > 0, st


# ---- 2. replay of a streaming run -----------------------------------------------------------------------------------
def test_replay_of_streaming_run():
    """Box-room scans streamed one bucket per lk_scan_update call (update_map = 1); the state and P each bucket ended with
    place that bucket's points in one lk_map_insert call on a second handle with the same starting map."""
    cfg, blob, _ = scenes.box_scene()
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    Q = abi.process_cov_Q(cfg)
    eng = _engine(cfg, blob)
    x, P = abi.default_states(1), abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE)
    clk["last_predict_time"], clk["last_update_time"] = 9.99, 9.985
    sets, rot, pos, rc, pc = [], [], [], [], []
    updated = 0
    for i in range(3):
        scan = sc.scan(rotvec=(0.0, 0.0, 0.01 * i), trans=(0.03 * i, -0.02 * i, 0.0), ext_R=R, ext_t=t, blind=cfg["blind"],
                       stream=880 + i, streaming=True, **mm.LIDAR)
        pts, offs, times = synth.bucketize(scan, begin_time=10.0 + 0.1 * i)
        for b in range(len(times)):
            p = pts[offs[b]:offs[b + 1]]
            out = eng.scan_update(x, P, Q, clk, p, [0, len(p)], times[b:b + 1], iters=1, update_map=True)
            updated += int(out["n_eff"][0] > 0)
            x, P, clk = out["x"], out["P"], out["clk"]
            Pm = P[0].reshape(30, 30)
            sets.append(p); rot.append(x["rot"][0]); pos.append(x["pos"][0]); rc.append(Pm[:3, :3]); pc.append(Pm[3:6, 3:6])
    assert updated > 100, updated
    twin = _engine(cfg, blob)
    twin.map_insert(np.concatenate(sets), mic.offsets([len(s) for s in sets]), rot, pos, rc, pc)
    n = exact(eng.map_download(), twin.map_download())
    print(f"[map insert] replay: buckets={len(sets)} updated={updated} nodes={n}")


# ---- 3. window boundaries -------------------------------------------------------------------------------------------
def test_window_boundaries():
    cfg = abi.CONFIGS["leg_fusion"]
    c = mic.room_trajectory(cfg, 48, 9700)
    pts, so = c["pts"], c["set_offsets"]
    assert len(pts) > 2 * WINDOW + 1000, len(pts)
    blob0 = mic.start_blob(cfg, c)
    whole = _engine(cfg, blob0)
    whole.map_insert(*mic.call(c))
    ref = whole.map_download()
    per_set = _engine(cfg, blob0)
    for s in range(len(so) - 1):
        per_set.map_insert(pts[so[s]:so[s + 1]], [0, so[s + 1] - so[s]], *(c[k][s:s + 1] for k in mic.CALL_KEYS[2:]))
    # arbitrary cuts, mid-set and across window boundaries, one call per piece
    cuts = np.unique(np.concatenate([[0, len(pts)], synth.rng(9710).integers(1, len(pts), 9), [WINDOW - 1, WINDOW + 1]]))
    pieces = _engine(cfg, blob0)
    for a, b in zip(cuts[:-1], cuts[1:]):
        s0 = int(np.searchsorted(so, a, side="right")) - 1
        s1 = int(np.searchsorted(so, b, side="left"))
        off = np.clip(so[s0:s1 + 1], a, b) - a
        pieces.map_insert(pts[a:b], off, *(c[k][s0:s1] for k in mic.CALL_KEYS[2:]))
    n1 = exact(ref, per_set.map_download())
    n2 = exact(ref, pieces.map_download())
    st = mapcmp.compare_blobs(mic.oracle_insert(cfg, blob0, *mic.call(c)), ref)
    print(f"[map insert] windows: points={len(pts)} nodes={n1}/{n2} planes={st['planes']}")


# ---- 4. hot images --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["room_on_blob", "room_empty", "cluttered"])
def test_hot_images_of_inserted_maps(name):
    cfg, c = mic.case(name)
    eng = _engine(cfg, mic.start_blob(cfg, c))
    eng.map_insert(*mic.call(c))
    x0 = gp.moving_state(c["rot"][0], c["pos"][0])
    if name == "cluttered":
        pts = c["pts"]
    else:
        sc = gp.map_cloud(cfg, mic.G, gp.G_POS)[0]
        pts = gp.room_scan(cfg, sc, 9820, False, n_az=900)
    r = mi._probe(eng, cfg, pts, x0)
    mi._report(f"map insert {name}", **r)
    assert r["ok"] > 1000, r


# ---- 5. storage -----------------------------------------------------------------------------------------------------
def test_freezes_and_cuts_recycle_tiles():
    cfg, c = mic.case("cluttered")
    eng = _engine(cfg)
    eng.map_insert(*mic.call(c))
    w = mm._walk(eng.map_download())
    mem = eng.map_memory()
    assert w["frozen"] > 10 and w["cut"] > 5, w
    # one standard tile back per frozen leaf and per cut node
    assert mem["free_point_slots"] >= mm._tile(cfg) * (w["frozen"] + w["cut"]) // 2, (mem, w)


def test_slide_between_calls_recycles_the_window():
    """The floor of test_gpu_map_memory inserted one scan per call at the pose it was taken from, sliding the map window
    between calls: once the window is full, new roots reuse what slid out and no pool grows."""
    cfg = mm.SLIDE_CFG
    eng, o, slide = _engine(cfg), lko_insert.Oracle(cfg), mm._OracleSlide(cfg)
    n, mem = 48, []
    for i in range(n):
        pos = np.array([mm.STEP_M * i, 0.0, 0.0])
        args = (mm._floor_scan(cfg, pos, i), [0, 2500], np.eye(3)[None], pos[None], 1e-6 * np.eye(3)[None], 1e-6 * np.eye(3)[None])
        eng.map_insert(*args)
        o.map_insert(*args)
        assert eng.map_slide(pos) == slide(o, pos)
        mem.append(eng.map_memory())
    last = 2 * n // 3
    for k in ("nodes", "point_slots"):
        per_scan = max(mem[i][k] - mem[i - 1][k] for i in range(1, n // 3))
        assert mem[-1][k] - mem[last][k] <= per_scan, (k, [m[k] for m in mem])
    assert mem[-1]["reallocs"] == mem[last]["reallocs"] and mem[-1]["free_nodes"] > 0, mem[-1]
    st = mapcmp.compare_blobs(o.map_export(), eng.map_download())
    assert st["planes"] > 500, st


def test_repeated_static_scene_stops_growing():
    """The same trajectory inserted again and again: its leaves fill up and freeze, their tiles are recycled, and no node
    or point slot is handed out after the first pass. (The headroom rule reserves a window's worst case above the bump
    pointer, so the pools may grow once more on the second pass, by half: ensure_headroom's growth step.)"""
    cfg, c = mic.case("room_on_blob")
    eng = _engine(cfg, mic.start_blob(cfg, c))
    mem = []
    for _ in range(6):
        eng.map_insert(*mic.call(c))
        mem.append(eng.map_memory())
    print("[map insert] repeated:", [(m["nodes"], m["point_slots"], m["pool_bytes"], m["reallocs"]) for m in mem])
    for m in mem[1:]:
        assert (m["nodes"], m["point_slots"]) == (mem[0]["nodes"], mem[0]["point_slots"]), mem
    for m in mem[2:]:
        assert (m["pool_bytes"], m["reallocs"]) == (mem[1]["pool_bytes"], mem[1]["reallocs"]), mem
    assert mem[-1]["free_point_slots"] > 0, mem


# ---- 6. host behaviour ----------------------------------------------------------------------------------------------
def test_staged_batch_survives_an_insert():
    cfg, blob, scans = scenes.box_scene()
    _, c = mic.case("cluttered")
    pts = scans[0]
    Q = abi.process_cov_Q(cfg)
    args = (abi.default_states(1), abi.init_cov(1), Q, np.zeros(1, abi.CLOCK_DTYPE), pts, [0, len(pts)], [0.0])
    # cluttered placed near the room's origin instead of at G, so that it touches the map the scan sees
    ins = (c["pts"], c["set_offsets"], np.tile(np.eye(3), (3, 1, 1)), np.zeros((3, 3)), c["rot_cov"], c["pos_cov"])
    a = _engine(cfg, blob)
    a.stage(*args)
    a.map_insert(*ins)
    a.run(iters=2)
    out_a = a.fetch()
    b = _engine(cfg, blob)
    b.map_insert(*ins)
    b.stage(*args)
    b.run(iters=2)
    out_b = b.fetch()
    assert out_a["n_eff"][0] > 1000
    for k in ("x", "P", "clk", "world", "n_eff"):
        x, y = np.asarray(out_a[k]), np.asarray(out_b[k])
        if x.dtype.names:
            x, y = x.view(np.float64), y.view(np.float64)
        np.testing.assert_array_equal(x, y, err_msg=k)


def _raw(eng, n_sets, pts, so, rot, pos, rc, pc):
    p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)  # noqa: E731
    return lib().lk_map_insert(eng.h, n_sets, p(pts), p(so), p(rot), p(pos), p(rc), p(pc))


def test_invalid_arguments_and_empty_calls():
    cfg, c = mic.case("room_empty")
    eng = _engine(cfg)
    eng.map_insert(*mic.call(c))
    before = eng.map_download()
    good = [np.ascontiguousarray(a, t) for a, t in zip(mic.call(c), (np.float32, np.uint32) + (np.float64,) * 4)]
    n = len(good[1]) - 1
    for i in range(6):
        bad = list(good)
        bad[i] = None
        assert _raw(eng, n, *bad) == -1, i
    so = good[1].copy()
    so[2] = so[1] - 1
    assert _raw(eng, n, good[0], so, *good[2:]) == -1
    for i in range(2, 6):
        for v in (np.nan, np.inf):
            bad = list(good)
            bad[i] = good[i].copy()
            bad[i].flat[len(bad[i].flat) // 2] = v
            assert _raw(eng, n, *bad) == -1, (i, v)
    assert _raw(eng, 0, None, None, None, None, None, None) == 0
    eng.map_insert(np.zeros((0, 4), np.float32), [0], np.zeros((0, 9)), np.zeros((0, 3)), np.zeros((0, 9)), np.zeros((0, 9)))
    exact(before, eng.map_download())
    with pytest.raises(LkError):
        eng.map_insert(c["pts"], c["set_offsets"], c["rot"], np.full((n, 3), np.nan), c["rot_cov"], c["pos_cov"])
