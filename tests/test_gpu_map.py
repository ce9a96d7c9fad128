"""Device-side map construction (BuildVoxelMap, init_plane, init/cut_octo_tree) against the oracle."""
import numpy as np
import pytest

import lko
import mapcmp
import scenes
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
# streaming scans with UpdateVoxelMap, device against the oracle
STATE_TOL = 7e-6  # (tests/scenes.py) worst measured on an H100 80GB HBM3: 7.0e-8 sd (the map built from an empty one)
COV_TOL = 4.5e-7  # worst measured: 4.6e-9


def _both(cfg, pw, pb, R=None, rot_cov=None, pos_cov=None):
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw, pb, R, rot_cov, pos_cov)
    eng = Engine(cfg)
    eng.map_build(pw, pb, R, rot_cov, pos_cov)
    return o.map_export(), eng.map_download(), eng


def test_build_planar_map_matches_oracle():
    cfg = abi.CONFIGS["leg_fusion"]
    R, t = abi.extrinsics(cfg)
    pw, pb = synth.planar_map_points(half_extent=10.0, ext_R=R, ext_t=t)
    a, b, eng = _both(cfg, pw, pb)
    st = mapcmp.compare_blobs(a, b)
    assert st["planes"] == 1600 and st["points"] == len(pw)
    s = eng.map_stats()
    assert s["roots"] == 1600 and s["planes"] == 1600 and s["points"] == len(pw)


def test_build_box_room_matches_oracle():
    cfg = abi.CONFIGS["diter"]
    R, t = abi.extrinsics(cfg)
    pw, pb = synth.BoxScene(ground_half_extent=18.0).map_points(ext_R=R, ext_t=t)
    a, b, _ = _both(cfg, pw, pb)
    st = mapcmp.compare_blobs(a, b)
    assert st["planes"] > 5000


def test_build_cluttered_scene_subdivides():
    """Dense non-planar clutter: roots fail the plane test, get cut into octants (2 layers),
    big leaves freeze (> max_points_num) — exercises cut_octo_tree and the freeze rules."""
    cfg = abi.CONFIGS["leg_fusion"]
    g = synth.rng(77)
    n = 60000
    pw = np.concatenate([
        g.uniform(-4, 4, (n // 2, 3)),                                   # volumetric clutter
        np.c_[g.uniform(-4, 4, (n // 4, 2)), 0.13 + 0.002 * g.standard_normal(n // 4)],  # a thin slab inside it
        g.uniform(4, 6, (n // 4, 3)) * np.array([1, 1, 0.05])]).astype(np.float32)
    pb = pw.copy()
    pb[:, 2] -= 0.2
    rot = synth.exp_so3([0.01, -0.02, 0.03])
    rc = np.diag([1e-6, 2e-6, 3e-6]); pc = np.diag([4e-6, 5e-6, 6e-6])
    a, b, _ = _both(cfg, pw, pb, rot, rc, pc)
    st = mapcmp.compare_blobs(a, b)
    assert st["interior"] > 100 and st["planes"] > 100


def test_map_upload_download_roundtrip():
    cfg, blob, _ = scenes.planar_scene(half_extent=6.0)
    eng = Engine(cfg)
    eng.map_upload(blob)
    st = mapcmp.compare_blobs(blob, eng.map_download(), rtol=1e-15)
    assert st["planes"] == 576


def _stream_case(streaming, iters=1, stream0=700, empty_map=False, n_scans=2, fast_insert=1, check_world=False, fused_insert=0):
    import test_gpu_parity as tp
    cfg, blob, scans = scenes.box_scene(batch=2, streaming=streaming, stream0=stream0)
    x0 = tp._moving_state() if streaming else abi.default_states(1)
    P0 = abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 9.99; clk["last_update_time"] = 9.985
    o = lko.Oracle(cfg)
    eng = Engine(cfg)
    eng.set_param("fast_insert", fast_insert)
    eng.set_param("fused_insert", fused_insert)
    if not empty_map:
        o.map_import(blob)
        eng.map_upload(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=iters, update_map=True)
    xg, Pg, cg = x0.copy(), P0.copy(), clk.copy()
    t0 = 10.0
    for s in scans[:n_scans]:  # two consecutive scans of one stream: the second one sees the map the first one left
        pts, offs, times = synth.bucketize(s, begin_time=t0)
        ro = o.process_scan(t0, pts)
        out = eng.scan_update(xg, Pg, abi.process_cov_Q(cfg), cg, pts, [0, len(pts)], times, scan_bucket_ptr=[0, len(times)],
                              bucket_offsets=offs, iters=iters, update_map=True)
        xo, Po, _, clko = o.get_filter()
        assert int(out["n_eff"][0]) == ro["n_eff"]
        scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL, f"scan at {t0:.1f}")
        if check_world:  # the re-projected cloud comes out of the insert's first phase on the fast path
            np.testing.assert_allclose(out["world"][:, :3], ro["world"][:, :3], rtol=0, atol=5e-6)
            np.testing.assert_array_equal(out["world"][:, 3], ro["world"][:, 3])
        xg, Pg, cg = out["x"], out["P"], out["clk"]
        t0 += 0.1
    # the device state differs from the oracle's by ~1e-11 relative, so do the inserted points
    st = mapcmp.compare_blobs(o.map_export(), eng.map_download(), rtol=1e-5, pt_atol=1e-8, var_rtol=1e-6)
    return st


def test_update_map_scan_at_once():
    """One bucket per scan: update, re-project, then UpdateVoxelMap of all ~28 k points (KILO.cc:215-231)."""
    st = _stream_case(streaming=False, check_world=True)
    assert st["planes"] > 3000


@pytest.mark.parametrize("insert", ["two-launch", "slice-and-sort", "in-kernel"])
@pytest.mark.parametrize("iters", [1, 2])
def test_update_map_streaming(iters, insert):
    """~50 buckets per scan, map mutated between buckets (refits every 6th insertion per leaf, freezes
    at 50 points, new roots / octants on demand) — the full reference loop on the device, through all three insert
    paths: two launches per small bucket, the general slice-and-sort path, and UpdateVoxelMap inside the persistent
    per-scan kernel (one launch per scan, grid barriers between the phases, map read through L2)."""
    st = _stream_case(streaming=True, iters=iters, fast_insert=0 if insert == "slice-and-sort" else 1, check_world=True,
                      fused_insert=1 if insert == "in-kernel" else 0)
    assert st["planes"] > 3000


def test_update_map_from_empty():
    """No prior map: the scan finds no residuals at first and only inserts (the map, roots included,
    is created by UpdateVoxelMap); later buckets of the same scan already match against it."""
    st = _stream_case(streaming=True, empty_map=True, stream0=900, n_scans=1)
    assert st["nodes"] > 3000 and st["points"] > 20000
    st = _stream_case(streaming=True, empty_map=True, stream0=900, n_scans=1, fused_insert=1)
    assert st["nodes"] > 3000 and st["points"] > 20000
