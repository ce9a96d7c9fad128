"""GPU parity: the CUDA path through the C ABI against the CPU oracle on identical inputs.
States are compared in posterior standard deviations and covariances in correlation units (scenes.state_err /
scenes.cov_err), so that the pose block is held to the same standard as the large imu_w / imu_a variances."""
import numpy as np
import pytest

import lko
import scenes
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
# (state_err, cov_err) tolerances, 100x the worst measured on an H100 80GB HBM3: 5.6e-11 sd (the throughput family, a 2 047-point scan,
# 2 iterations) and 1.7e-14 with a static map; 2.1e-9 sd and 4.0e-12 for the streaming fixture with UpdateVoxelMap
STATE_TOL = 5e-9
COV_TOL = 1e-12
MAP_STATE_TOL = 2e-7
MAP_COV_TOL = 4e-10


def _oracle_bucket(cfg, blob, pts, x0, P0, iters=1, gain=lko.GAIN_INFORMATION, t=0.0):
    o = lko.Oracle(cfg)
    o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE))
    o.set_options(gain_mode=gain, iters=iters, update_map=False)
    r = o.predict_update_point(t, pts, debug=True)
    x, P, _, clk = o.get_filter()
    return r, x, P, clk


def test_config1_planar_literal_pin():
    """BASELINE config 1: 2 048-pt planar scan, identity prior, 1 iteration, oracle in the
    reference's literal measurement-space (N x N) form."""
    cfg, blob, pts = scenes.planar_scene()
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    ro, xo, Po, clko = _oracle_bucket(cfg, blob, pts, x0, P0, gain=lko.GAIN_LITERAL)
    eng = Engine(cfg)
    eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), pts, [0, len(pts)], [0.0])
    assert int(out["n_eff"][0]) == ro["n_eff"] > 0.9 * len(pts)
    scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL)
    np.testing.assert_allclose(out["world"][:, :3], ro["world"][:, :3], rtol=0, atol=2e-6)
    assert np.all(out["world"][:, 3] == 255.0)
    assert out["clk"]["last_update_time"][0] == clko["last_update_time"][0]


def _check_debug_rows(n):
    cfg, blob, pts = scenes.planar_scene(n=n, seed_stream=7)
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    ro, _, _, _ = _oracle_bucket(cfg, blob, pts, x0, P0)
    eng = Engine(cfg)
    eng.map_upload(blob)
    d = eng.debug_residuals(x0, P0, pts)
    assert np.array_equal(d["key"], ro["key"])
    assert np.array_equal(d["ok"], ro["ok"])
    m = ro["ok"].astype(bool)
    # eigenvector sign is free: compare sign-invariant products
    np.testing.assert_allclose(d["h"][m] * d["z"][m, None], ro["h"][m] * ro["z"][m, None], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(d["R"][m], ro["R"][m], rtol=1e-9)


def test_debug_rows_match_oracle():
    _check_debug_rows(1500)


def test_debug_rows_match_oracle_sliced_chunks():
    """One bucket above 132 x 256 points gets 3 840-point chunks, which the debug kernel walks in 256-point slices."""
    _check_debug_rows(40000)


@pytest.mark.parametrize("iters", [1, 3])
def test_box_room_batch(iters):
    cfg, blob, scans = scenes.box_scene(batch=3)
    eng = Engine(cfg)
    eng.map_upload(blob)
    x0 = abi.default_states(3); P0 = abi.init_cov(3)
    pts = np.concatenate(scans)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(3, abi.CLOCK_DTYPE), pts, offs, np.zeros(3), iters=iters)
    for i, s in enumerate(scans):
        ro, xo, Po, _ = _oracle_bucket(cfg, blob, s, x0[i:i + 1], P0[i:i + 1], iters=iters)
        assert int(out["n_eff"][i]) == ro["n_eff"] > 0
        scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, STATE_TOL, COV_TOL, f"scan {i}")


@pytest.mark.parametrize("fused", [0, 1])
def test_single_scan_paths_agree_with_oracle(fused):
    """batch = 1 runs go through the persistent per-scan kernel (fused=1) or the multi-kernel path
    (fused=0); both must match the oracle and — same arithmetic, same order — each other bitwise."""
    cfg, blob, scans = scenes.box_scene(batch=1, stream0=300)
    eng = Engine(cfg)
    eng.set_param("fused", fused)
    eng.map_upload(blob)
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), scans[0], [0, len(scans[0])], [0.0], iters=3)
    ro, xo, Po, _ = _oracle_bucket(cfg, blob, scans[0], x0, P0, iters=3)
    assert int(out["n_eff"][0]) == ro["n_eff"] > 0
    scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL)
    np.testing.assert_allclose(out["world"][:, :3], ro["world"][:, :3], rtol=0, atol=2e-6)
    key = "_single_scan_ref"
    if key in globals():
        np.testing.assert_array_equal(globals()[key]["x"].view(np.float64), out["x"].view(np.float64))
        np.testing.assert_array_equal(globals()[key]["P"], out["P"])
    globals()[key] = out


def test_throughput_family_chunk_edges():
    """Calls with >= 2 scans take the throughput family: 3 840- / 256-point chunks, warps streaming 32-point groups
    through a software pipeline. Scan lengths sit on every edge of that machinery (one point, group and chunk
    boundaries +-1, several chunks, a warp without work); the kernel must reproduce the oracle's residual counts
    exactly and its state / covariance within tolerance, whatever mixture of lengths shares the call."""
    ws = 2
    cfg, blob, scans = scenes.box_scene(batch=2, lidar=synth.OS64)
    base = np.concatenate(scans)
    assert len(base) > 8000
    sizes = [1, 31, 32, 33, 255, 256, 257, 1919, 1920, 1921, 2047, 2048, 2049, 3839, 3840, 3841, 7777]
    rs = np.random.default_rng(5)
    pieces = []
    for n in sizes:
        o = int(rs.integers(0, len(base) - n))
        pieces.append(base[o:o + n].copy())
    B = len(pieces)
    pts = np.concatenate(pieces)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in pieces])]).astype(np.uint32)
    x0 = abi.default_states(B); P0 = abi.init_cov(B)
    eng = Engine(cfg)
    eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(B, abi.CLOCK_DTYPE), pts, offs, np.zeros(B), iters=2)
    again = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(B, abi.CLOCK_DTYPE), pts, offs, np.zeros(B), iters=2)
    np.testing.assert_array_equal(out["P"], again["P"])  # run-to-run bitwise
    np.testing.assert_array_equal(out["x"].view(np.float64), again["x"].view(np.float64))
    some = 0
    for i, s in enumerate(pieces):
        ro, xo, Po, _ = _oracle_bucket(cfg, blob, s, x0[i:i + 1], P0[i:i + 1], iters=2)
        assert int(out["n_eff"][i]) == ro["n_eff"], (ws, len(s))
        if ro["n_eff"] > 0:
            some += 1
            scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, STATE_TOL, COV_TOL, f"{len(s)} points")
        np.testing.assert_allclose(out["world"][offs[i]:offs[i + 1], :3], ro["world"][:, :3], rtol=0, atol=5e-6)
    assert some >= len(sizes) - 3
    # many small scans: more chunks than SMs, so the persistent variant walks several chunks per block (stage ring
    # re-used across chunk and scan boundaries) and the others run several waves
    sizes2 = [int(v) for v in rs.integers(260, 700, size=220)]
    pieces2 = []
    for n in sizes2:
        o = int(rs.integers(0, len(base) - n))
        pieces2.append(base[o:o + n].copy())
    B2 = len(pieces2)
    pts2 = np.concatenate(pieces2)
    offs2 = np.concatenate([[0], np.cumsum(sizes2)]).astype(np.uint32)
    x2 = abi.default_states(B2); P2 = abi.init_cov(B2)
    out2 = eng.scan_update(x2, P2, abi.process_cov_Q(cfg), np.zeros(B2, abi.CLOCK_DTYPE), pts2, offs2, np.zeros(B2), iters=2,
                           want_world=False)
    for i in range(0, B2, 7):
        ro, xo, Po, _ = _oracle_bucket(cfg, blob, pieces2[i], x2[i:i + 1], P2[i:i + 1], iters=2)
        assert int(out2["n_eff"][i]) == ro["n_eff"], (ws, i)
        if ro["n_eff"] > 0:
            scenes.check_filter(out2["x"][i:i + 1], out2["P"][i], xo, Po, STATE_TOL, COV_TOL, f"scan {i} of {B2}")


@pytest.mark.parametrize("streaming", [False, True])
def test_direct_io_matches_staged_bitwise(streaming):
    """One scan through lk_scan_update with page-locked caller buffers runs in direct mode (points read in
    place, world cloud / filter stored in place, small inputs in the kernel parameter block). Same kernel, same
    arithmetic: every output must equal the staged path's bit for bit."""
    cfg, blob, scans = scenes.box_scene(batch=1, streaming=streaming, stream0=300)
    if streaming:
        pts, offs, times = synth.bucketize(scans[0], begin_time=100.0)
        x0 = _moving_state()
        clk0 = np.zeros(1, abi.CLOCK_DTYPE); clk0["last_predict_time"] = 99.99; clk0["last_update_time"] = 99.985
    else:
        pts, offs, times = scans[0], np.array([0, len(scans[0])], np.uint32), np.zeros(1)
        x0 = abi.default_states(1); clk0 = np.zeros(1, abi.CLOCK_DTYPE)
    P0 = abi.init_cov(1); Q = abi.process_cov_Q(cfg)
    eng = Engine(cfg)
    eng.map_upload(blob)
    kw = dict(scan_bucket_ptr=[0, len(times)], bucket_offsets=offs, iters=2)
    outs = {}
    for name, params, pinned in (("staged", dict(direct_io=0), True), ("pageable", dict(direct_io=1), False),
                                 ("direct", dict(direct_io=1, inline_in=0), True), ("direct+inline", dict(direct_io=1, inline_in=1), True)):
        for k, v in params.items():
            eng.set_param(k, v)
        outs[name] = eng.scan_update(x0, P0, Q, clk0, pts, [0, len(pts)], times, pinned=pinned, **kw)
        # a second call re-uses the cached process noise
        again = eng.scan_update(x0, P0, Q, clk0, pts, [0, len(pts)], times, pinned=pinned, **kw)
        np.testing.assert_array_equal(again["P"], outs[name]["P"])
    ref = outs["staged"]
    assert int(ref["n_eff"][0]) > 0
    for name, o in outs.items():
        np.testing.assert_array_equal(o["x"].view(np.float64), ref["x"].view(np.float64), err_msg=name)
        np.testing.assert_array_equal(o["P"], ref["P"], err_msg=name)
        np.testing.assert_array_equal(o["clk"].view(np.float64), ref["clk"].view(np.float64), err_msg=name)
        np.testing.assert_array_equal(o["n_eff"], ref["n_eff"], err_msg=name)
        np.testing.assert_array_equal(np.asarray(o["world"]), np.asarray(ref["world"]), err_msg=name)
    # a changed process noise must be picked up by the cached copy
    Q2 = Q * 2.0
    eng.set_param("direct_io", 1); eng.set_param("inline_in", 1)
    a = eng.scan_update(x0, P0, Q2, clk0, pts, [0, len(pts)], times, pinned=True, **kw)
    eng.set_param("direct_io", 0)
    b = eng.scan_update(x0, P0, Q2, clk0, pts, [0, len(pts)], times, pinned=True, **kw)
    eng.set_param("direct_io", 1)
    np.testing.assert_array_equal(a["P"], b["P"])
    if streaming:
        assert not np.array_equal(a["P"], ref["P"])


def _oracle_stream(cfg, blob, pts_sorted, begin_time, x0, P0, clk0, iters=1, update_map=False, gain=lko.GAIN_INFORMATION,
                   imu=None, kin=None, imu_mode_only=True):
    o = lko.Oracle(cfg)
    o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk0)
    o.set_options(gain_mode=gain, iters=iters, update_map=update_map, imu_mode_only=imu_mode_only)
    r = o.process_scan(begin_time, pts_sorted, imu=imu, kin=kin)
    x, P, _, clk = o.get_filter()
    return r, x, P, clk, o


def _moving_state():
    """A prior with non-trivial velocity / angular rate / acceleration so that predict matters."""
    x0 = abi.default_states(1)
    x0["vel"][0] = (0.4, -0.2, 0.05)
    x0["imu_w"][0] = (0.02, -0.03, 0.15)
    x0["imu_a"][0] = (0.3, 0.1, 9.7)
    x0["ba"][0] = (0.01, -0.02, 0.03)
    x0["bw"][0] = (1e-3, 2e-3, -1e-3)
    return x0


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("iters", [1, 2])
def test_streaming_buckets_static_map(fused, iters):
    """~50 time buckets per scan (2 ms quantisation): predict (eskf.cc:83-89) -> residuals -> update per
    bucket, map static. Exercises rows a1, a2, a8, a9, a10 through both device paths."""
    cfg, blob, scans = scenes.box_scene(batch=1, streaming=True, stream0=500)
    pts, offs, times = synth.bucketize(scans[0], begin_time=100.0)
    assert len(times) > 30
    x0 = _moving_state(); P0 = abi.init_cov(1)
    clk0 = np.zeros(1, abi.CLOCK_DTYPE); clk0["last_predict_time"] = 99.99; clk0["last_update_time"] = 99.985
    ro, xo, Po, clko, _ = _oracle_stream(cfg, blob, pts, 100.0, x0, P0, clk0, iters=iters)
    eng = Engine(cfg)
    eng.set_param("fused", fused)
    eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), clk0, pts, [0, len(pts)], times, scan_bucket_ptr=[0, len(times)],
                          bucket_offsets=offs, iters=iters)
    assert int(out["n_eff"][0]) == ro["n_eff"] > 0
    scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL)
    assert out["clk"]["last_predict_time"][0] == clko["last_predict_time"][0]
    assert out["clk"]["last_update_time"][0] == clko["last_update_time"][0]
    np.testing.assert_allclose(out["world"][:, :3], ro["world"][:, :3], rtol=0, atol=5e-6)
    np.testing.assert_array_equal(out["world"][:, 3], ro["world"][:, 3])


def test_golden_fixtures_on_gpu():
    """The committed fixtures (tests/golden/, made by make_golden.py from the oracle in the build
    container) replayed on the device: config 1, and one streaming scan with map updates."""
    import os
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    g = np.load(os.path.join(gdir, "config1_planar.npz"))
    cfg, blob, pts = scenes.planar_scene()
    assert np.array_equal(pts, g["pts"])
    x0 = abi.default_states(1); P0 = abi.init_cov(1)
    eng = Engine(cfg); eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), np.zeros(1, abi.CLOCK_DTYPE), pts, [0, len(pts)], [0.0])
    xg = g["x"].view(abi.STATE_DTYPE)
    assert int(out["n_eff"][0]) == int(g["n_eff"])
    scenes.check_filter(out["x"], out["P"][0], xg, g["P"], STATE_TOL, COV_TOL, "config1_planar")

    g = np.load(os.path.join(gdir, "streaming_box.npz"))
    cfg, blob, scans = scenes.box_scene(batch=1, streaming=True, stream0=700, ground_half_extent=12.0)
    pts, offs, times = synth.bucketize(scans[0], begin_time=10.0)
    x0 = g["x0"].view(abi.STATE_DTYPE); P0 = abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 9.99; clk["last_update_time"] = 9.985
    eng = Engine(cfg); eng.map_upload(blob)
    out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), clk, pts, [0, len(pts)], times, scan_bucket_ptr=[0, len(times)],
                          bucket_offsets=offs, update_map=True)
    assert int(out["n_eff"][0]) == int(g["n_eff"])
    scenes.check_filter(out["x"], out["P"][0], g["x"].view(abi.STATE_DTYPE), g["P"], MAP_STATE_TOL, MAP_COV_TOL, "streaming_box")
    np.testing.assert_array_equal(out["clk"].view(np.float64), g["clk"])
    st = eng.map_stats()
    assert st["roots"] == int(g["n_roots"]) and st["nodes"] >= int(g["n_nodes"]) and st["points"] == int(g["n_points"])
    assert st["planes"] == int(g["n_planes"])


def test_batched_results_do_not_depend_on_sharding():
    """SURVEY §4 multi-GPU invariant: per-scan outputs are bitwise identical however a batch is cut into
    shards (chunking is a function of the bucket alone, partial sums are added in a fixed order, and every
    batch of >= 2 scans runs the same kernel family) — and identical from run to run."""
    from legkilo_b200 import shard
    cfg, blob, scans = scenes.box_scene(batch=4, stream0=1300)
    eng = Engine(cfg); eng.map_upload(blob)
    x0 = abi.default_states(4); P0 = abi.init_cov(4); clk = np.zeros(4, abi.CLOCK_DTYPE); Q = abi.process_cov_Q(cfg)
    pts = np.concatenate(scans)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.uint32)
    full = eng.scan_update(x0, P0, Q, clk, pts, offs, np.zeros(4), iters=3)
    again = eng.scan_update(x0, P0, Q, clk, pts, offs, np.zeros(4), iters=3)
    assert full["x"].tobytes() == again["x"].tobytes() and full["P"].tobytes() == again["P"].tobytes()
    for rank in range(2):
        s = shard.shard_batch(rank, 2, x0, P0, clk, pts, offs, np.zeros(4))
        part = eng.scan_update(s["x"], s["P"], Q, s["clk"], s["pts"], s["scan_offsets"], s["bucket_times"], iters=3)
        assert part["x"].tobytes() == full["x"][s["lo"]:s["hi"]].tobytes()
        assert part["P"].tobytes() == full["P"][s["lo"]:s["hi"]].tobytes()
        assert np.array_equal(part["n_eff"], full["n_eff"][s["lo"]:s["hi"]])
