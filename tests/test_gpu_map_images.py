"""The hot plane images (lk_device.cuh: HotRec) of maps that the device built, updated, slid and recycled itself.

Every call whose map stays fixed for the call evaluates the root planes on these 144-byte images, not on the node
records. The images are written in several places: k_hot_from_nodes after an upload, hot_after_fit after every plane fit
of the bulk build and of the inserts (both branches), node_reset for new roots and child groups and for the octrees a slide
drops, and the node-pool growth copy. Each scenario below brings a map into the state its name says (and asserts, from
downloads and counters, that it got there), then probes it (_probe):

a. lk_debug_residuals in both forms, the hot images (default) and the node records (knob "debug_records"), against the
   CPU oracle fed the downloaded blob;
b. the two forms against each other: h, z bitwise; rows that come out of an octree descent (node records in both forms)
   bitwise in every field; R of root planes within the rounding of the collapsed sigma_plane;
c. static lk_scan_update calls (per-scan kernel, multi-kernel path, the scan twice in one call = throughput family)
   against the oracle, and the per-scan kernel bitwise against the multi-kernel path;
d. a second handle fed the downloaded blob, whose images k_hot_from_nodes rebuilds: bitwise every output of b and c.
"""
import numpy as np
import pytest

import lko
import scenes
import test_gpu_map_memory as mm
import test_gpu_parity as tp
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
STATE_TOL = 2.4e-11  # (tests/scenes.py) worst measured on an H100 80GB HBM3 (here and in test_gpu_map_insert.py): 2.4e-13 sd
COV_TOL = 1.3e-10  # worst measured: 1.3e-12
ITERS = 2
PROBE_LIDAR = dict(n_rings=16, n_az=900, fov_deg=(-15.0, 15.0))  # ~14 000 points: one 256-point chunk per block
# the insert paths of update_map calls: (fast_insert, fused_insert)
INSERT_PATHS = {"two-launch": (1, 0), "slice-and-sort": (0, 0), "in-kernel": (1, 1)}


# ---- map inspection --------------------------------------------------------------------------------------------------
def _walk(blob):
    """Per node of the download: reachable from a root, the key of that root, and the node's layer."""
    _, roots, nodes, _, _ = abi.parse_map_blob(blob)
    reach = np.zeros(len(nodes), bool)
    rkey = np.zeros((len(nodes), 3), np.int64)
    stack = [(int(r["node"]), tuple(int(k) for k in r["key"])) for r in roots]
    while stack:
        i, k = stack.pop()
        reach[i] = True
        rkey[i] = k
        f = int(nodes[i]["flags"])
        for c in range(8):
            if (f >> abi.NODE_CHILDMASK_SHIFT) & (1 << c):
                stack.append((int(nodes[i]["child_base"]) + c, k))
    layer = (nodes["flags"].astype(np.int64) >> abi.NODE_LAYER_SHIFT) & 0xff
    return reach, rkey, layer


def _is_plane(nodes):
    return (nodes["flags"] & abi.NODE_IS_PLANE) != 0


def _code(keys):
    k = np.asarray(keys, np.int64) + (1 << 20)
    return (k[..., 0] << 42) | (k[..., 1] << 21) | k[..., 2]


def _root_nodes(blob, keys):
    """node of the root under each key (-1: no root there)."""
    _, roots, _, _, _ = abi.parse_map_blob(blob)
    rc = _code(roots["key"])
    order = np.argsort(rc)
    q = _code(keys)
    at = np.clip(np.searchsorted(rc[order], q), 0, max(len(rc) - 1, 0))
    hit = (rc[order][at] == q) if len(rc) else np.zeros(len(q), bool)
    out = np.full(len(q), -1, np.int64)
    out[hit] = roots["node"][order][at][hit]
    return out


def _root_flags(blob, keys):
    """flags of the root under each key (-1: no root there)."""
    nd = _root_nodes(blob, keys)
    out = np.full(len(nd), -1, np.int64)
    out[nd >= 0] = abi.parse_map_blob(blob)[2]["flags"][nd[nd >= 0]]
    return out


def _sigma_terms(blob, cfg, x, pts, keys):
    """Per point, the largest |J| |Sigma_plane| |J|^T (J = [pw - c, -n]) over the root planes of its voxel and of the 26
    around it: the size of the terms that sum to sigma_plane, so a small multiple of eps times it bounds how differently
    the collapsed form of the hot image and the 21-term form of the node record can round."""
    _, _, nodes, _, _ = abi.parse_map_blob(blob)
    Re, te = abi.extrinsics(cfg)
    pw = (pts[:, :3].astype(np.float64) @ Re.T + te) @ x["rot"][0].reshape(3, 3).T + x["pos"][0]
    iu = np.triu_indices(6)
    out = np.zeros(len(pts))
    for d in np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3):
        nd = _root_nodes(blob, keys + d)
        at = np.flatnonzero(nd >= 0)
        at = at[_is_plane(nodes[nd[at]])]
        N = nodes[nd[at]]
        S = np.zeros((len(at), 6, 6))
        S[:, iu[0], iu[1]] = np.abs(N["plane_var"])
        S[:, iu[1], iu[0]] = np.abs(N["plane_var"])
        J = np.abs(np.concatenate([pw[at] - N["center"], N["normal"]], 1))
        out[at] = np.maximum(out[at], np.einsum("ni,nij,nj->n", J, S, J))
    return out


def _no_root_plane_near(blob, keys):
    """True where neither the voxel of `key` nor any of its 26 neighbours is a root that holds a plane: a row there can
    only have come out of an octree descent (the one neighbour the reference falls back to is among the 26)."""
    clear = np.ones(len(keys), bool)
    for d in np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3):
        f = _root_flags(blob, keys + d)
        clear &= ~((f >= 0) & ((f & abi.NODE_IS_PLANE) != 0))
    return clear


def _body_pts(cfg, pw, pos=(0.0, 0.0, 0.0)):
    R, t = abi.extrinsics(cfg)
    pts = np.zeros((len(pw), 4), np.float32)
    pts[:, :3] = synth.world_to_body(np.asarray(pw, float), np.eye(3), np.asarray(pos, float), R, t).astype(np.float32)
    return pts


def _on_planes(blob, idx, per, rs, noise=0.002):
    """`per` world points on each plane node in `idx`: within its radius (at most 0.1 m) of the centre, `noise` off."""
    _, _, nodes, _, _ = abi.parse_map_blob(blob)
    out = []
    for i in idx:
        c, n = nodes[i]["center"], nodes[i]["normal"]
        e1 = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(n, e1)
        r = min(float(nodes[i]["radius"]), 0.1)
        u, v = rs.uniform(-r, r, per), rs.uniform(-r, r, per)
        out.append(c + u[:, None] * e1 + v[:, None] * e2 + noise * rs.standard_normal(per)[:, None] * n)
    return np.concatenate(out) if out else np.zeros((0, 3))


def _child_planes(blob):
    """Plane nodes of layer >= 1 under roots that hold no plane."""
    nodes = abi.parse_map_blob(blob)[2]
    reach, _, layer = _walk(blob)
    return np.flatnonzero(reach & _is_plane(nodes) & (layer >= 1))


def _changes(a, b):
    """What happened to the nodes of download `a` by download `b` (same node index, same root key)."""
    _, ra, na, _, _ = abi.parse_map_blob(a)
    _, rb, nb, _, _ = abi.parse_map_blob(b)
    reach_a, key_a, _ = _walk(a)
    reach_b, key_b, _ = _walk(b)
    m = len(na)
    same = reach_a & reach_b[:m] & np.all(key_a == key_b[:m], axis=1)
    pa, pb = _is_plane(na), _is_plane(nb[:m])
    refit = same & pa & pb & np.any(na["center"] != nb[:m]["center"], axis=1)
    flip = same & pa & ~pb
    new_roots = len(set(_code(rb["key"]).tolist()) - set(_code(ra["key"]).tolist()))
    return dict(refits=int(refit.sum()), flips=int(flip.sum()), new_roots=new_roots, flipped=np.flatnonzero(flip))


# ---- the probe -------------------------------------------------------------------------------------------------------
def _rows(eng, x0, P0, pts, records):
    eng.set_param("debug_records", records)
    try:
        return eng.debug_residuals(x0, P0, pts)
    finally:
        eng.set_param("debug_records", 0)


def _static(eng, cfg, pts, x0, P0):
    """The map stays fixed: the per-scan kernel (fused = 1), the multi-kernel path (fused = 0), and the scan twice in one
    call (the throughput family and its fallback kernel)."""
    Q = abi.process_cov_Q(cfg)
    n = len(pts)
    out = {}
    for fused in (1, 0):
        eng.set_param("fused", fused)
        out[fused] = eng.scan_update(x0, P0, Q, np.zeros(1, abi.CLOCK_DTYPE), pts, [0, n], [0.0], iters=ITERS)
    eng.set_param("fused", 1)
    out[2] = eng.scan_update(np.concatenate([x0, x0]), np.concatenate([P0, P0]), Q, np.zeros(2, abi.CLOCK_DTYPE),
                             np.concatenate([pts, pts]), [0, n, 2 * n], [0.0, 0.0], iters=ITERS)
    return out


def _same(a, b, what):
    for k in a:
        if a[k] is None:
            continue
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype.names:
            x, y = x.view(np.float64), y.view(np.float64)
        np.testing.assert_array_equal(x, y, err_msg=f"{what}: {k}")


def _probe(eng, cfg, pts, x0, P0=None):
    """a-d of the module docstring on the map `eng` holds. Returns row counts."""
    P0 = abi.init_cov(1) if P0 is None else np.asarray(P0).reshape(1, 900)
    blob = eng.map_download()
    hot, rec = _rows(eng, x0, P0, pts, 0), _rows(eng, x0, P0, pts, 1)
    # a. both forms against the oracle on the exact blob
    ro, _, _, _ = tp._oracle_bucket(cfg, blob, pts, x0, P0)
    m = ro["ok"].astype(bool)
    for name, d in (("hot", hot), ("records", rec)):
        np.testing.assert_array_equal(d["key"], ro["key"], err_msg=name)
        np.testing.assert_array_equal(d["ok"], ro["ok"], err_msg=name)
        np.testing.assert_allclose(d["h"][m] * d["z"][m, None], ro["h"][m] * ro["z"][m, None], rtol=1e-9, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(d["R"][m], ro["R"][m], rtol=1e-9, err_msg=name)
    # b. hot images against node records: sigma_plane is the only thing the two forms compute differently
    np.testing.assert_array_equal(hot["h"], rec["h"])
    np.testing.assert_array_equal(hot["z"], rec["z"])
    descent = m & _no_root_plane_near(blob, hot["key"])
    np.testing.assert_array_equal(hot["R"][descent], rec["R"][descent])
    # R = ratio (sigma_plane + body): the two forms may differ by the rounding of sigma_plane alone. That is ~1e-16 of R on
    # a well-conditioned plane, and up to eps times the size of its terms on a plane fit from a few points, whose
    # plane_var reaches 1e3 and whose sigma_plane is a cancellation of terms thousands of times larger
    dR = np.abs(hot["R"][m] - rec["R"][m])
    bound = cfg["lidar_point_meas_ratio"] * 32 * np.finfo(float).eps * _sigma_terms(blob, cfg, x0, pts[m], hot["key"][m])
    assert np.all(dR <= bound), (dR / bound).max()
    # c. static calls against the oracle, per-scan kernel bitwise the multi-kernel path
    st = _static(eng, cfg, pts, x0, P0)
    ro2, xo, Po, _ = tp._oracle_bucket(cfg, blob, pts, x0, P0, iters=ITERS)
    for k, out in st.items():
        for i in range(len(out["x"])):
            assert int(out["n_eff"][i]) == ro2["n_eff"], (k, i, out["n_eff"], ro2["n_eff"])
            if ro2["n_eff"] == 0:
                continue
            scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, STATE_TOL, COV_TOL, f"fused {k} scan {i}")
    _same({k: st[1][k] for k in ("x", "P", "n_eff")}, st[0], "fused 1 vs 0")
    # d. a second handle whose images come from k_hot_from_nodes: every output bitwise
    twin = Engine(cfg)
    twin.map_upload(blob)
    _same(hot, _rows(twin, x0, P0, pts, 0), "twin hot rows")
    _same(rec, _rows(twin, x0, P0, pts, 1), "twin record rows")
    st2 = _static(twin, cfg, pts, x0, P0)
    for k in st:
        _same(st[k], st2[k], f"twin static {k}")
    twin.close()
    home = _root_flags(blob, hot["key"])
    return dict(ok=int(m.sum()), home_no_plane=int((m & (home >= 0) & ((home & abi.NODE_IS_PLANE) == 0)).sum()),
                descent=int(descent.sum()), n_eff=int(ro2["n_eff"]))


def _room_scan(cfg, sc, i, rotvec=(0.0, 0.0, 0.0), trans=(0.0, 0.0, 0.0), lidar=PROBE_LIDAR, streaming=False):
    R, t = abi.extrinsics(cfg)
    return sc.scan(rotvec=rotvec, trans=trans, ext_R=R, ext_t=t, blind=cfg["blind"], stream=i, streaming=streaming, **lidar)


def _report(name, **kv):
    print(f"[map images] {name}: " + " ".join(f"{k}={v}" for k, v in kv.items()))


# ---- 1. device bulk build --------------------------------------------------------------------------------------------
def test_bulk_build_box_room():
    """The box room with a shelf in it: two boards 0.25 m apart across 4 x 4 m. A voxel that holds both boards is no plane
    (its smallest eigenvalue is ~0.016), so it is cut, and each of its octants holds a piece of one board: a plane."""
    cfg = abi.CONFIGS["diter"]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=18.0)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    rs = synth.rng(804)
    n = 40 * 8 * 8 * 2
    shelf = np.c_[rs.uniform(2.0, 6.0, (n, 2)), np.where(np.arange(n) % 2 == 0, 0.125, 0.375) + 0.005 * rs.standard_normal(n)]
    eng = Engine(cfg)
    eng.map_build(np.concatenate([pw, shelf.astype(np.float32)]), np.concatenate([pb, _body_pts(cfg, shelf)[:, :3]]))
    blob = eng.map_download()
    kids = _child_planes(blob)
    assert len(kids) > 400, len(kids)
    x0 = abi.default_states(1)
    x0["pos"][0] = (0.01, -0.02, 0.01)
    pts = np.concatenate([_room_scan(cfg, sc, 801, rotvec=(0.002, -0.001, 0.003), trans=(0.01, -0.02, 0.01)),
                          _body_pts(cfg, _on_planes(blob, kids, 3, synth.rng(802)), x0["pos"][0])])
    r = _probe(eng, cfg, pts, x0)
    _report("bulk build, box room", child_planes=len(kids), **r)
    assert r["home_no_plane"] > 1000 and r["descent"] > 1000, r


def test_bulk_build_cluttered_scene():
    """The scene of test_gpu_map.test_build_cluttered_scene_subdivides: roots of volumetric clutter cut into octants (few of
    which hold a plane), leaves frozen at build. Probed on points of the child planes, of the clutter and of the slab."""
    cfg = abi.CONFIGS["leg_fusion"]
    g = synth.rng(77)
    n = 60000
    pw = np.concatenate([
        g.uniform(-4, 4, (n // 2, 3)),
        np.c_[g.uniform(-4, 4, (n // 4, 2)), 0.13 + 0.002 * g.standard_normal(n // 4)],
        g.uniform(4, 6, (n // 4, 3)) * np.array([1, 1, 0.05])]).astype(np.float32)
    pb = pw.copy()
    pb[:, 2] -= 0.2
    rot = synth.exp_so3([0.01, -0.02, 0.03])
    eng = Engine(cfg)
    eng.map_build(pw, pb, rot, np.diag([1e-6, 2e-6, 3e-6]), np.diag([4e-6, 5e-6, 6e-6]))
    blob = eng.map_download()
    kids = _child_planes(blob)
    w = mm._walk(blob)
    assert len(kids) > 0 and w["cut"] > 100 and w["frozen"] > 100, (len(kids), w)
    rs = synth.rng(803)
    world = np.concatenate([_on_planes(blob, kids, 20, rs), rs.uniform(-4, 4, (6000, 3)),
                            np.c_[rs.uniform(-4, 4, (2000, 2)), 0.13 + 0.002 * rs.standard_normal(2000)]])
    r = _probe(eng, cfg, _body_pts(cfg, world), abi.default_states(1))
    _report("bulk build, cluttered", child_planes=len(kids), cut=w["cut"], frozen=w["frozen"], **r)
    assert r["home_no_plane"] > 0, r


# ---- 2. streaming inserts --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def box_blob():
    cfg, blob, _ = scenes.box_scene()
    return cfg, blob


def _stream(cfg, blob, path):
    s = mm._Stream(cfg, blob, oracle=False)
    fast, fused = INSERT_PATHS[path]
    s.eng.set_param("fast_insert", fast)
    s.eng.set_param("fused_insert", fused)
    return s


@pytest.mark.parametrize("start", ["uploaded", "empty"])
@pytest.mark.parametrize("path", list(INSERT_PATHS))
def test_streaming_inserts(box_blob, path, start):
    """Three streaming scans with update_map through one insert path, from an uploaded map or from an empty handle; probed
    after the first and after the last. The last scans are twice the size of the first, so the pools grow between the
    probes (lk_api.cu reserves per scanned point)."""
    cfg, blob = box_blob
    s = _stream(cfg, blob if start == "uploaded" else None, path)
    sc = synth.BoxScene(ground_half_extent=20.0)
    downloads, mem = [], []
    for i in range(3):
        lidar = mm.LIDAR if i == 0 else dict(mm.LIDAR, n_rings=16)
        pose = dict(rotvec=(0.0, 0.0, 0.01 * i), trans=(0.03 * i, -0.02 * i, 0.0))
        s.step(_room_scan(cfg, sc, 810 + i, lidar=lidar, streaming=True, **pose))
        if i in (0, 2):
            downloads.append(s.eng.map_download())
            mem.append(s.eng.map_memory())
            r = _probe(s.eng, cfg, _room_scan(cfg, sc, 820 + i, **pose), s.x, s.P)
            assert r["ok"] > 200, r
    ch = _changes(downloads[0], downloads[1])
    _report(f"stream {path} from {start}", reallocs=(mem[0]["reallocs"], mem[1]["reallocs"]),
            **{k: v for k, v in ch.items() if k != "flipped"}, **r)
    assert ch["refits"] > 0 and ch["new_roots"] > 0, ch
    assert mem[1]["reallocs"] > mem[0]["reallocs"], mem


@pytest.mark.parametrize("path", list(INSERT_PATHS))
def test_refit_turns_a_plane_into_no_plane(path):
    """A root that holds a flat patch of six points takes points from two sheets at the top and the bottom of its voxel:
    the refit on the sixth new point fails the planarity test, the root holds no plane any more, and its hot image must say
    so (hot_after_fit's radius = -1 branch), or the patch's plane keeps producing rows."""
    cfg = abi.CONFIGS["leg_fusion"]
    rs = synth.rng(830)
    # corners and edge midpoints of voxel (0, 0, -2): every layout below spreads ~0.2 m along x and y
    xy = np.array([[0.05, 0.05], [0.45, 0.05], [0.05, 0.45], [0.45, 0.45], [0.25, 0.05], [0.25, 0.45]])
    patch = np.c_[xy, np.full(6, -0.75)]
    o = lko.Oracle(cfg)
    o.build_voxel_map(patch.astype(np.float32), _body_pts(cfg, patch)[:, :3])
    blob = o.map_export()
    _, roots, nodes, _, _ = abi.parse_map_blob(blob)
    assert len(roots) == 1 and _is_plane(nodes).all()
    # the refit on the sixth new point sees the patch and 6 points 0.22 m above or below it, uncorrelated with x and y: its
    # smallest eigenvalue is 0.023, the planarity threshold 0.01
    dz = 0.22 * np.array([1, -1, -1, 1, 1, 1])
    sheets = np.c_[np.vstack([xy, xy]), -0.75 + np.r_[dz, -dz]]
    s = _stream(cfg, blob, path)
    probe = _body_pts(cfg, np.c_[rs.uniform(0.02, 0.48, (400, 2)), -0.75 + 0.002 * rs.standard_normal(400)])
    x0 = abi.default_states(1)
    before = s.eng.map_download()
    r0 = _probe(s.eng, cfg, probe, x0)
    assert r0["ok"] > 300, r0
    s.step(_body_pts(cfg, sheets))
    after = s.eng.map_download()
    ch = _changes(before, after)
    assert ch["flips"] == 1 and list(ch["flipped"]) == [int(roots[0]["node"])], ch
    r1 = _probe(s.eng, cfg, probe, x0)
    _report(f"plane -> no plane, {path}", flips=ch["flips"], rows_before=r0["ok"], rows_after=r1["ok"])
    assert r1["ok"] == 0, r1


# ---- 3. freeze -------------------------------------------------------------------------------------------------------
def test_frozen_leaves(box_blob):
    """Dense streaming scans until leaves reach max_points_num and freeze; probed where the frozen planes are."""
    cfg, blob = box_blob
    s = _stream(cfg, blob, "two-launch")
    sc = synth.BoxScene(ground_half_extent=20.0)
    for i in range(3):
        s.step(_room_scan(cfg, sc, 840 + i, lidar=synth.VLP16, streaming=True, trans=(0.02 * i, 0.0, 0.0)))
    down = s.eng.map_download()
    frozen = mm._walk(down)["frozen"]
    assert frozen > 50, frozen
    _, roots, nodes, _, _ = abi.parse_map_blob(down)
    f = nodes["flags"][roots["node"]]
    frozen_roots = roots["key"][(f & abi.NODE_IS_PLANE != 0) & (f & abi.NODE_UPDATE_ENABLE == 0)]
    pts = _room_scan(cfg, sc, 850, trans=(0.04, 0.0, 0.0))
    r = _probe(s.eng, cfg, pts, s.x, s.P)
    d = s.eng.debug_residuals(s.x, np.asarray(s.P).reshape(1, 900), pts)
    on_frozen = int((d["ok"].astype(bool) & np.isin(_code(d["key"]), _code(frozen_roots))).sum())
    _report("frozen", frozen=frozen, frozen_roots=len(frozen_roots), rows_on_frozen=on_frozen, **r)
    assert on_frozen > 100, on_frozen


# ---- 4. slide and recycle --------------------------------------------------------------------------------------------
def test_slide_recycled_roots():
    """The floor of test_gpu_map_memory driven until roots dropped by a slide come back as the nodes of new roots. A
    recycled root's hot image must show its own plane (or none), never the one of the root that slid out."""
    cfg = mm.SLIDE_CFG
    s = mm._Stream(cfg, oracle=False)
    owner = {}  # node -> key of the plane root that held it in an earlier download
    recycled = []
    for i in range(40):
        pos = (mm.STEP_M * i, 0.0, 0.0)
        s.step(mm._floor_scan(cfg, pos, i), pos=pos)
        down = s.eng.map_download()
        _, roots, nodes, _, _ = abi.parse_map_blob(down)
        recycled = [(tuple(int(v) for v in r["key"]), int(r["node"])) for r in roots
                    if int(r["node"]) in owner and owner[int(r["node"])] != tuple(int(v) for v in r["key"])]
        if len(recycled) >= 20:
            break
        for r in roots:
            if _is_plane(nodes[int(r["node"])]):
                owner[int(r["node"])] = tuple(int(v) for v in r["key"])
        s.eng.map_slide(pos)
    assert len(recycled) >= 20, (i, len(recycled))
    mem = s.eng.map_memory()
    keys = np.array([k for k, _ in recycled])
    fl = nodes["flags"][[n for _, n in recycled]]
    # points of the floor on every recycled root and on its 8 neighbours, plus a scan from where the robot stands
    rs = synth.rng(860)
    v = cfg["voxel_size"]
    world = []
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            base = (keys[:, :2] + (dx, dy)) * v
            for _ in range(3):
                world.append(np.c_[base + rs.uniform(0.02, v - 0.02, base.shape), -0.75 + 0.003 * rs.standard_normal(len(base))])
    world = np.concatenate(world)
    x0 = abi.default_states(1)
    x0["pos"][0] = pos
    pts = np.concatenate([_body_pts(cfg, world, pos), mm._floor_scan(cfg, pos, 1000 + i)])
    r = _probe(s.eng, cfg, pts, x0)
    _report("slide", scans=i + 1, recycled_roots=len(recycled), recycled_planes=int(((fl & abi.NODE_IS_PLANE) != 0).sum()),
            free_nodes=mem["free_nodes"], **r)
    assert r["ok"] > 1000, r


# ---- 5. dense plane covariances ----------------------------------------------------------------------------------------
def _dense_blob(blob, seed, zero_cross=False):
    """Every plane node of `blob` gets a random dense SPD plane_var (L L^T) with a strong correlation between the block that
    multiplies pw - c and the block that multiplies the normal; centre, normal, d and radius are kept. Scaled so that
    sigma_plane is of the order of the body and state terms (~1e-3)."""
    hd, roots, nodes, aux, pts = abi.parse_map_blob(blob)
    nodes = nodes.copy()
    rs = synth.rng(seed)
    iu = np.triu_indices(6)
    scale = np.sqrt(np.array([1e-2] * 3 + [1e-3] * 3) / 6.0)
    for i in np.flatnonzero(_is_plane(nodes)):
        A = rs.standard_normal((3, 6))
        Q, _ = np.linalg.qr(rs.standard_normal((3, 3)))
        L = np.vstack([A, Q @ A + 0.5 * rs.standard_normal((3, 6))])
        S = (L @ L.T) * np.outer(scale, scale)
        if zero_cross:
            S[:3, 3:] = 0.0
            S[3:, :3] = 0.0
        nodes[i]["plane_var"] = S[iu]
    return abi.make_map_blob(roots, nodes, aux, pts)


def test_dense_plane_covariances(box_blob):
    cfg, blob = box_blob
    sc = synth.BoxScene(ground_half_extent=20.0)
    x0 = abi.default_states(1)
    pts = _room_scan(cfg, sc, 870, rotvec=(0.002, -0.001, 0.003), trans=(0.01, -0.02, 0.01))
    res = {}
    for zero in (False, True):
        eng = Engine(cfg)
        eng.map_upload(_dense_blob(blob, 871, zero_cross=zero))
        r = _probe(eng, cfg, pts, x0)
        res[zero] = (r, eng.debug_residuals(x0, abi.init_cov(1), pts))
        eng.close()
    (r, d), (_, dz) = res[False], res[True]
    m = d["ok"].astype(bool) & dz["ok"].astype(bool)
    moved = np.abs(d["R"][m] - dz["R"][m]) / np.abs(d["R"][m]) > 1e-6
    _report("dense covariances", moved=f"{int(moved.sum())}/{int(m.sum())}", **r)
    assert r["ok"] > 5000 and moved.mean() > 0.8, (r, moved.mean())
