"""Recycled map storage: frozen leaves, cut parents and slid-out octrees give their point tiles and nodes back to the
map's free lists, so a long streaming run stops growing its pools (lk_map_memory) while computing exactly what it did."""
import numpy as np
import pytest

import lko
import mapcmp
import scenes
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
# one streaming scan with UpdateVoxelMap from a common prior, device against the oracle
STATE_TOL = 4.8e-4  # (tests/scenes.py) worst measured on an H100 80GB HBM3: 4.9e-6 sd, a scan into a map of frozen leaves
COV_TOL = 3.9e-6  # worst measured: 4.0e-8

LIDAR = dict(n_rings=8, n_az=450, fov_deg=(-15.0, 15.0))  # ~3 000 points per revolution, 50 buckets of 2 ms
N_FROZEN = 200


def _tile(cfg):
    return (cfg["max_points_num"] + 2 + 1) & ~1  # the standard tile: even_up(max_points_num + 2)


class _Stream:
    """One device handle (and optionally the oracle) fed the same scans. Every scan starts the oracle from the device's
    filter, so the per-scan comparison does not depend on how far the run has gone."""

    def __init__(self, cfg, blob=None, fused_insert=0, oracle=True):
        self.cfg = cfg
        self.Q = abi.process_cov_Q(cfg)
        self.eng = Engine(cfg)
        self.eng.set_param("fused_insert", fused_insert)
        self.o = lko.Oracle(cfg) if oracle else None
        if self.o is not None:
            self.o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=True)
        if blob is not None:
            self.eng.map_upload(blob)
            if self.o is not None:
                self.o.map_import(blob)
        self.x = abi.default_states(1)
        self.x0 = self.x.copy()
        self.P = abi.init_cov(1)
        self.clk = np.zeros(1, abi.CLOCK_DTYPE)
        self.clk["last_predict_time"] = 9.99
        self.clk["last_update_time"] = 9.985
        self.t0 = 10.0

    def step(self, scan, pos=None):
        if pos is not None:
            # the pose the scan was taken from as the prior, at rest, with the initial covariance: the floor alone fixes
            # neither x, y nor yaw, so the filter would drift there and its covariance would grow without bound
            self.x = abi.default_states(1)
            self.x["pos"][0] = pos
            self.x["imu_a"][0] = (0.0, 0.0, 9.81)  # cancels gravity in the prediction
            self.P = abi.init_cov(1)
        pts, offs, times = synth.bucketize(scan, begin_time=self.t0)
        out = self.eng.scan_update(self.x, self.P, self.Q, self.clk, pts, [0, len(pts)], times, scan_bucket_ptr=[0, len(times)],
                                   bucket_offsets=offs, iters=1, update_map=True)
        if self.o is not None:
            self.o.set_filter(self.x, self.P, self.Q, self.clk)
            ro = self.o.process_scan(self.t0, pts)
            xo, Po, _, _ = self.o.get_filter()
            assert int(out["n_eff"][0]) == ro["n_eff"]
            scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL, f"scan at {self.t0:.1f}")
        self.x, self.P, self.clk = out["x"], out["P"], out["clk"]
        self.t0 += 0.1
        return out


def _walk(blob):
    """Nodes reachable from the root keys: (frozen, cut, can still take points, non-standard slots held)."""
    _, roots, nodes, aux, _ = abi.parse_map_blob(blob)
    seen = set()
    stack = [int(r["node"]) for r in roots]
    while stack:
        i = stack.pop()
        seen.add(i)
        f = int(nodes[i]["flags"])
        for c in range(8):
            if (f >> abi.NODE_CHILDMASK_SHIFT) & (1 << c):
                stack.append(int(nodes[i]["child_base"]) + c)
    idx = np.fromiter(seen, np.int64, len(seen))
    f = nodes["flags"][idx].astype(np.int64)
    init = (f & abi.NODE_INIT_OCTO) != 0
    frozen = init & ((f & abi.NODE_UPDATE_ENABLE) == 0)
    cut = init & ((f & abi.NODE_IS_PLANE) == 0) & (((f >> abi.NODE_CHILDMASK_SHIFT) & 0xff) != 0)
    return dict(frozen=int(frozen.sum()), cut=int(cut.sum()), growable=int((~frozen & ~cut).sum()), caps=aux["pts_cap"])


@pytest.fixture(scope="module")
def frozen_run():
    """~200 scans of the box room from a slowly moving pose: many leaves reach max_points_num and freeze."""
    cfg, blob, _ = scenes.box_scene()
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=20.0)
    s = _Stream(cfg, blob)
    scans, outs, mem, blobs = [], [], [], {}
    for i in range(N_FROZEN):
        scan = sc.scan(rotvec=(0.0, 0.0, 0.002 * i), trans=(0.004 * i, -0.002 * i, 0.0), ext_R=R, ext_t=t, blind=cfg["blind"],
                       stream=500 + i, streaming=True, **LIDAR)
        scans.append(scan)
        outs.append(s.step(scan))
        mem.append(s.eng.map_memory())
        if i + 1 in (N_FROZEN // 2, N_FROZEN):
            blobs[i + 1] = s.eng.map_download()
    return dict(cfg=cfg, blob=blob, scans=scans, outs=outs, mem=mem, blobs=blobs, oracle_map=s.o.map_export())


def test_frozen_leaves_return_their_tiles(frozen_run):
    r = frozen_run
    cfg, mem, blobs = r["cfg"], r["mem"], r["blobs"]
    tile = _tile(cfg)
    end, mid = _walk(blobs[N_FROZEN]), _walk(blobs[N_FROZEN // 2])
    assert end["frozen"] > 200
    m = mem[-1]
    held = m["point_slots"] - m["free_point_slots"]
    # one standard tile per node that can still take points, plus the bump blocks above the standard size; before
    # recycling every frozen leaf and cut parent kept its tile on top of this
    nonstd = int(end["caps"][end["caps"] > tile].sum())
    assert held <= tile * end["growable"] + nonstd, (held, end, nonstd)
    assert m["free_point_slots"] > 0
    freed = tile * (end["frozen"] + end["cut"] - mid["frozen"] - mid["cut"])
    grown = m["point_slots"] - mem[N_FROZEN // 2 - 1]["point_slots"]
    assert freed > 0 and grown < freed, (grown, freed)
    # 200 scans' worth of points, each inserted with a state ~1e-11 (relative) off the oracle's: centres drift by ~1e-8 m
    st = mapcmp.compare_blobs(r["oracle_map"], blobs[N_FROZEN], rtol=1e-5, pt_atol=1e-6, var_rtol=1e-6)
    assert st["planes"] > 3000


def test_in_kernel_insert_recycles_the_same_way(frozen_run):
    """The frozen-leaf stream with UpdateVoxelMap inside the persistent per-scan kernel: bitwise the per-bucket path."""
    r = frozen_run
    s = _Stream(r["cfg"], r["blob"], fused_insert=1, oracle=False)
    for scan, ref in zip(r["scans"], r["outs"]):
        out = s.step(scan)
        for k in ("x", "clk"):
            np.testing.assert_array_equal(out[k].view(np.float64), ref[k].view(np.float64))
        for k in ("P", "n_eff", "world"):
            np.testing.assert_array_equal(out[k], ref[k])
    assert s.eng.map_memory()["free_point_slots"] > 0
    mapcmp.compare_blobs(r["blobs"][N_FROZEN], s.eng.map_download(), rtol=1e-15, pt_atol=0.0, var_rtol=0.0)


# ---- sliding window over a long floor ------------------------------------------------------------------------------
SLIDE_CFG = dict(abi.CONFIGS["leg_fusion"], half_map_size=16, sliding_thresh=2.0)  # window of +-16 voxels = +-8 m
STEP_M = 0.9  # metres per scan along x


def _floor_scan(cfg, pos, i, n=2500, radius=7.0, z=-0.75, sigma=0.01):
    """`n` points of the floor z = const within `radius` of `pos`, in the body frame of a LiDAR there (identity attitude),
    all in one bucket: a bucket of a spinning LiDAR sees a narrow wedge of a bare floor, which leaves roll / pitch loose."""
    R, t = abi.extrinsics(cfg)
    g = synth.rng(900 + i)
    r = np.sqrt(g.uniform(1.0, radius * radius, n))
    a = g.uniform(0.0, 2 * np.pi, n)
    pw = np.stack([pos[0] + r * np.cos(a), pos[1] + r * np.sin(a), z + sigma * g.standard_normal(n)], 1)
    pb = synth.world_to_body(pw, np.eye(3), np.asarray(pos, float), R, t)
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = pb.astype(np.float32)
    return pts


class _OracleSlide:
    """mapSliding on the oracle's map (voxel_map.cc:552-594): export, drop the roots outside the window, import."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.last = np.zeros(3)

    def __call__(self, o, pos):
        pos = np.asarray(pos, float)
        if np.linalg.norm(pos - self.last) < self.cfg["sliding_thresh"]:
            return False, 0
        self.last = pos.copy()
        k = np.floor(pos / self.cfg["voxel_size"]).astype(np.int64)
        h = self.cfg["half_map_size"]
        _, roots, nodes, aux, pts = abi.parse_map_blob(o.map_export())
        keep = np.all((roots["key"] >= k - h) & (roots["key"] <= k + h), axis=1)
        o.map_import(abi.make_map_blob(roots[keep], nodes, aux, pts))
        return True, int((~keep).sum())


def _slide_run(n_scans, oracle=True, stop=None):
    s = _Stream(SLIDE_CFG, oracle=oracle)
    slide = _OracleSlide(SLIDE_CFG)
    mem = []
    for i in range(n_scans):
        pos = (STEP_M * i, 0.0, 0.0)
        s.step(_floor_scan(SLIDE_CFG, pos, i), pos=pos)
        slid, removed = s.eng.map_slide(pos)
        if oracle:
            assert (slid, removed) == slide(s.o, pos)
        mem.append(s.eng.map_memory())
        if stop is not None and stop(i, slid, mem[-1]):
            break
    return s, mem


def test_slide_recycles_the_window():
    """Drive 43 m over a long floor, sliding the map window (+-8 m) after every scan: once the window is full, every
    new root reuses the node and the tile of one that slid out, and no pool grows any more."""
    n = 48
    s, mem = _slide_run(n)
    last = 2 * n // 3
    for k in ("nodes", "point_slots"):
        # one scan's worth: the largest growth of a single scan while the window fills (the first scan builds the map)
        per_scan = max(mem[i][k] - mem[i - 1][k] for i in range(1, n // 3))
        grown = mem[-1][k] - mem[last][k]
        assert grown <= per_scan, (k, grown, per_scan, [m[k] for m in mem])
    assert mem[-1]["reallocs"] == mem[last]["reallocs"]
    assert mem[-1]["free_nodes"] > 0
    st = mapcmp.compare_blobs(s.o.map_export(), s.eng.map_download(), rtol=1e-5, pt_atol=1e-8, var_rtol=1e-6)
    assert st["planes"] > 500


def test_blob_right_after_a_slide_round_trips():
    """A download taken while recycled entries sit on the free lists uploads into a fresh handle, and both handles then
    compute bitwise the same."""
    s, mem = _slide_run(40, oracle=False, stop=lambda i, slid, m: i >= 12 and slid and m["free_nodes"] > 0
                        and m["free_point_slots"] > 0)
    assert mem[-1]["free_nodes"] > 0 and len(mem) < 40
    a = s.eng.map_download()
    other = _Stream(SLIDE_CFG, blob=a, oracle=False)
    mapcmp.compare_blobs(a, other.eng.map_download(), rtol=1e-15)
    other.x, other.P, other.clk, other.t0 = s.x.copy(), s.P.copy(), s.clk.copy(), s.t0
    i0 = len(mem)
    for i in range(i0, i0 + 6):
        pos = (STEP_M * i, 0.0, 0.0)
        scan = _floor_scan(SLIDE_CFG, pos, i)
        out_a, out_b = s.step(scan, pos=pos), other.step(scan, pos=pos)
        for k in ("x", "clk"):
            np.testing.assert_array_equal(out_a[k].view(np.float64), out_b[k].view(np.float64))
        for k in ("P", "n_eff", "world"):
            np.testing.assert_array_equal(out_a[k], out_b[k])
    mapcmp.compare_blobs(s.eng.map_download(), other.eng.map_download(), rtol=1e-15, pt_atol=0.0, var_rtol=0.0)
