"""The device at general priors: a map built from a rotated, off-origin first frame, priors composed from it, dense SPD
covariances (optionally with a skew part), per-scan priors and clocks in a batch, a scene kilometres from the origin.
Every other device test starts from an identity attitude at the origin with P0 = 1e-6 I, where a transposed rotation, a
swapped or misplaced covariance block, a transposed P, a dropped row of K or one scan's prior read for all give the same
numbers. Oracle: tests/test_general_prior.py pins it to the reference at such priors."""
import os

import numpy as np
import pytest

import general_prior as gp
import lko
import mapcmp
import scenes
from legkilo_b200 import Engine, abi, shard, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G = synth.exp_so3(gp.G_ROTVEC)
# (state_err, cov_err) tolerances (tests/scenes.py), each 100x the worst measured on an H100 80GB HBM3:
# - the device (information form) against the oracle in the same form, static map: 6.7e-12 sd, 2.9e-14;
# - heterogeneous batches, whose streaming scans carry absolute stamps of 1.7e9 s: 1.6e-9 sd, 2.5e-11;
# - the reference-made bucket fixtures (literal gain, with UpdateVoxelMap): 4.2e-8 sd, 9.9e-12.
STATE_TOL = 6e-10
COV_TOL = 2.9e-12
HETERO_TOLS = (1.5e-7, 2.5e-9)
FIXTURE_TOLS = (4e-6, 9e-10)


def _load(name):
    d = dict(np.load(os.path.join(GOLD, name)))
    for k in ("x0", "x"):
        d[k] = d[k].view(abi.STATE_DTYPE)
    for k in ("clk0", "clk"):
        d[k] = d[k].view(abi.CLOCK_DTYPE)
    return d


def _check_fixture(d, x, P, clk, world, n_eff, blob, tols, center_atol, map_rtol=1e-5, d_atol=1e-5, radius_rtol=1e-6):
    assert int(n_eff) == int(d["n_eff"]) > 0
    scenes.check_filter(x, P, d["x"], d["P"], *tols)
    assert np.asarray(clk).tobytes() == d["clk"].tobytes()
    err = np.abs(world[:, :3] - d["world"][:, :3])
    assert (err <= gp.world_atol(d["world"])).all(), err.max()
    np.testing.assert_array_equal(world[:, 3], d["world"][:, 3])
    st = mapcmp.compare_digest(d["map1"], blob, rtol=map_rtol, center_atol=center_atol, d_atol=d_atol, radius_rtol=radius_rtol)
    assert st["planes"] > 100


def _engine(cfg, pw, pb, **params):
    eng = Engine(cfg)
    for k, v in params.items():
        eng.set_param(k, v)
    rot_cov, pos_cov = gp.map_covs(G)
    eng.map_build(pw, pb, R=G, rot_cov=rot_cov, pos_cov=pos_cov)
    return eng


def _oracle_map(cfg, pos):
    sc, pw, pb = gp.map_cloud(cfg, G, pos)
    o = lko.Oracle(cfg)
    rot_cov, pos_cov = gp.map_covs(G)
    o.build_voxel_map(pw, pb, R=G, rot_cov=rot_cov, pos_cov=pos_cov)
    return sc, o.map_export()


def _oracle_bucket(cfg, blob, pts, x0, P0, clk0, t, iters=1, debug=False):
    o = lko.Oracle(cfg)
    o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk0)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=iters, update_map=False)
    r = o.predict_update_point(t, pts, debug=debug)
    x, P, _, clk = o.get_filter()
    return r, x, P, clk


def _oracle_stream(cfg, blob, pts, begin, x0, P0, clk0, iters=1):
    o = lko.Oracle(cfg)
    o.map_import(blob)
    o.set_filter(x0, P0, abi.process_cov_Q(cfg), clk0)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=iters, update_map=False)
    r = o.process_scan(begin, pts)
    x, P, _, clk = o.get_filter()
    return r, x, P, clk


# ---- 1. the reference-made fixtures on every device path ------------------------------------------------------------------

BUCKET_PATHS = [("fused", dict(fused=1), False), ("multi-kernel", dict(fused=0), False), ("insert-in-kernel", dict(fused_insert=1), False),
                ("direct", dict(direct_io=1, inline_in=0), True), ("direct+inline", dict(direct_io=1, inline_in=1), True)]


@pytest.mark.parametrize("name", ["leg_fusion", "hilti", "asym", "far"])
@pytest.mark.parametrize("path,params,pinned", BUCKET_PATHS, ids=[p[0] for p in BUCKET_PATHS])
def test_bucket_fixture_on_device_paths(name, path, params, pinned):
    d = _load(f"ref_general_bucket_{name}.npz")
    cfg = abi.CONFIGS["hilti" if name == "hilti" else "leg_fusion"]
    eng = _engine(cfg, d["pw"], d["pb"], **params)
    scale = max(1.0, np.abs(d["pw"]).max() / 100)
    # BuildVoxelMap forms a plane's covariance as sum(p p^T) / N - c c^T (voxel_map.cc:49-54). Kilometres from the origin
    # that cancels terms ~1e9 times the spread of a small plane, so the device's summation order moves radius and
    # plane_var by up to ~1e-6 there (1e-16 at the other fixtures); the tolerances grow with the distance.
    far = 1.0 if scale < 10 else 100.0
    mapcmp.compare_digest(d["map0"], eng.map_download(), rtol=1e-6 * far, center_atol=1e-10 * scale, radius_rtol=1e-6 * far)
    if far > 1.0:
        # Those plane differences move this bucket's update by ~2e-4 of its step, so the far replay starts from the
        # oracle's BuildVoxelMap (equal to the reference's to 1e-7, tests/test_general_prior.py) uploaded to the device.
        rot_cov, pos_cov = gp.map_covs(G)
        o = lko.Oracle(cfg)
        o.build_voxel_map(d["pw"], d["pb"], R=G, rot_cov=rot_cov, pos_cov=pos_cov)
        eng.map_upload(o.map_export())
    n = len(d["pts"])
    out = eng.scan_update(d["x0"], d["P0"], abi.process_cov_Q(cfg), d["clk0"], d["pts"], [0, n], [float(d["t"])], iters=1,
                          update_map=True, pinned=pinned)
    _check_fixture(d, out["x"], out["P"][0], out["clk"], np.asarray(out["world"]), out["n_eff"][0], eng.map_download(), FIXTURE_TOLS,
                   1e-8 * scale, map_rtol=1e-5 * far, radius_rtol=1e-6 * far)


@pytest.mark.parametrize("kind", ["imu", "kin"])
@pytest.mark.parametrize("insert", ["per-bucket", "in-kernel"])
def test_stream_fixture_process_scan(kind, insert):
    d = _load(f"ref_general_stream_{kind}.npz")
    cfg = abi.CONFIGS["leg_fusion"]
    meas = d["meas"].view(abi.IMU_DTYPE if kind == "imu" else abi.KINIMU_DTYPE)
    eng = _engine(cfg, d["pw"], d["pb"], fused_insert=1 if insert == "in-kernel" else 0)
    pts, offs, times = synth.bucketize(d["pts"], begin_time=float(d["begin"]))
    assert pts.tobytes() == d["pts"].tobytes()
    out = eng.process_scan(d["x0"], d["P0"], abi.process_cov_Q(cfg), d["clk0"], pts, offs, times, imu=meas if kind == "imu" else None,
                           kin=meas if kind == "kin" else None, gravity=9.81, acc_norm=9.79, iters=1, update_map=True)
    _check_fixture(d, out["x"], out["P"], out["clk"], out["world"], out["n_eff"], eng.map_download(), gp.STREAM_TOLS, 1e-6,
                   map_rtol=1e-4, d_atol=1e-3)


# ---- 2. per-point rows at the general prior ---------------------------------------------------------------------------------

def _scene_for_rows(pos, stream=9400):
    cfg = abi.CONFIGS["leg_fusion"]
    sc, blob = _oracle_map(cfg, pos)
    pts = gp.room_scan(cfg, sc, stream, False, n_rings=16, n_az=360)
    g = synth.rng(stream + 50)
    return cfg, blob, pts, gp.prior_at(G, pos, g), gp.dense_cov(g)


def _rows_match(eng, cfg, blob, pts, x0, P0):
    ro, _, _, _ = _oracle_bucket(cfg, blob, pts, x0, P0, np.zeros(1, abi.CLOCK_DTYPE), 0.0, debug=True)
    d = eng.debug_residuals(x0, P0, pts)
    assert np.array_equal(d["key"], ro["key"])
    assert np.array_equal(d["ok"], ro["ok"]), np.flatnonzero(d["ok"] != ro["ok"])
    m = ro["ok"].astype(bool)
    assert m.sum() > 0.5 * len(pts)
    # z is the float dis_to_plane_: far from the origin s = n.pw + d cancels km-sized terms, and a rounding of s one way
    # or the other can move z by one float ulp
    zulp = np.spacing(np.abs(ro["z"][m]).astype(np.float32)).astype(np.float64)
    np.testing.assert_array_less(np.abs(d["h"][m] * d["z"][m, None] - ro["h"][m] * ro["z"][m, None]),
                                 1e-9 * np.abs(ro["h"][m] * ro["z"][m, None]) + np.abs(ro["h"][m]) * zulp[:, None] + 1e-12)
    np.testing.assert_allclose(d["R"][m], ro["R"][m], rtol=1e-9)
    return ro


@pytest.mark.parametrize("records", [0, 1])
def test_debug_rows_at_general_prior(records):
    cfg, blob, pts, x0, P0 = _scene_for_rows(gp.G_POS)
    eng = Engine(cfg)
    eng.set_param("debug_records", records)
    eng.map_upload(blob)
    ro = _rows_match(eng, cfg, blob, pts, x0, P0)
    assert (ro["key"] < 0).any()
    # the state term decides the gate here: the same points and pose at P = 1e-6 I give another set of rows
    riso = _rows_match(eng, cfg, blob, pts, x0, abi.init_cov(1))
    flips = int((ro["ok"] != riso["ok"]).sum())
    print(f"gate decisions changed by the state term: {flips} of {len(pts)}")
    assert flips > 0
    # and so does the skewed covariance (its symmetric part is what the gate reads)
    _rows_match(eng, cfg, blob, pts, x0, gp.skewed(P0, synth.rng(9401)))


# ---- 3. static and streaming scan_update against the oracle ------------------------------------------------------------------

@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("streaming", [False, True])
@pytest.mark.parametrize("iters", [1, 3])
def test_scan_update_against_oracle(iters, streaming, asym):
    cfg = abi.CONFIGS["leg_fusion"]
    sc, blob = _oracle_map(cfg, gp.G_POS)
    g = synth.rng(9500 + 2 * streaming)
    x0 = gp.prior_at(G, gp.G_POS, g)
    P0 = gp.dense_cov(g)
    if asym:
        P0 = gp.skewed(P0, g)
    clk0 = np.zeros(1, abi.CLOCK_DTYPE); clk0["last_predict_time"] = 99.99; clk0["last_update_time"] = 99.985
    scan = gp.room_scan(cfg, sc, 9510, streaming, n_rings=16, n_az=240)
    if streaming:
        pts, offs, times = synth.bucketize(scan, begin_time=100.0)
        assert len(times) > 30
        ro, xo, Po, clko = _oracle_stream(cfg, blob, pts, 100.0, x0, P0, clk0, iters=iters)
        kw = dict(scan_bucket_ptr=[0, len(times)], bucket_offsets=offs)
    else:
        pts, times = scan, np.array([100.0])
        ro, xo, Po, clko = _oracle_bucket(cfg, blob, pts, x0, P0, clk0, 100.0, iters=iters)
        kw = {}
        # rows 6..29 of K are reached: the update moves vel, ba and bw by a visible fraction of the pose step
        _, xp, _, _ = _oracle_bucket(cfg, blob, pts[:0], x0, P0, clk0, 100.0)
        dx = lko.boxminus(xo, xp)
        pose, rest = np.abs(dx[:6]).max(), np.abs(dx[6:15]).reshape(3, 3).max(axis=1)
        print(f"update step: pose {pose:.3e}, vel / ba / bw {rest}")
        assert (rest > 1e-3 * pose).all()
    outs = {}
    for fused in (1, 0):
        eng = Engine(cfg)
        eng.set_param("fused", fused)
        eng.map_upload(blob)
        out = eng.scan_update(x0, P0, abi.process_cov_Q(cfg), clk0, pts, [0, len(pts)], times, iters=iters, **kw)
        assert int(out["n_eff"][0]) == ro["n_eff"] > 0
        scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL, f"fused {fused}")
        np.testing.assert_array_equal(out["clk"].view(np.float64), clko.view(np.float64))
        err = np.abs(out["world"][:, :3] - ro["world"][:, :3])
        assert (err <= gp.world_atol(ro["world"])).all(), err.max()
        outs[fused] = out
    for k in ("x", "P", "clk", "n_eff", "world"):
        assert np.asarray(outs[0][k]).tobytes() == np.asarray(outs[1][k]).tobytes(), k


# ---- 4. heterogeneous batches in the throughput family ---------------------------------------------------------------------

SIZES = [1, 31, 32, 33, 255, 256, 257, 1919, 1920, 1921, 2047, 2048, 2049, 3839, 3840, 3841, 7777]


def _rotated_cov(g, scale):
    """A dense P0 whose attitude / position blocks (and their cross blocks) are turned by a random rotation."""
    P = gp.dense_cov(g, scale=scale).reshape(30, 30)
    T = np.eye(30)
    Rr = gp.so3_uniform(g)
    T[:3, :3] = Rr; T[3:6, 3:6] = Rr
    return (T @ P @ T.T).ravel()


def _hetero_batch(streaming):
    """B scans on the chunk-edge sizes, each from its own pose with its own prior, P0 (scaled, rotated), clock and time
    base. Scan 1 repeats scan 0's points from another prior."""
    cfg = abi.CONFIGS["leg_fusion"]
    sc, blob = _oracle_map(cfg, gp.G_POS)
    g = synth.rng(9600 + streaming)
    B = len(SIZES)
    x0 = np.zeros(B, abi.STATE_DTYPE); P0 = np.zeros((B, 900)); clk = np.zeros(B, abi.CLOCK_DTYPE)
    pieces, bo, bt, sbp = [], [0], [], [0]
    for i, n in enumerate(SIZES):
        rv = synth.exp_so3([0, 0, g.uniform(0, 2 * np.pi)]) @ synth.exp_so3(2e-3 * g.standard_normal(3))
        trans = g.uniform(-0.5, 0.5, 3) * (1, 1, 0.1)
        if i == 1:
            piece = pieces[0][:, :].copy()
        else:
            scan = gp.room_scan(cfg, sc, 9610 + i, streaming, rotvec=lko.log_so3(rv), trans=trans, n_rings=32, n_az=512)
            o = int(g.integers(0, len(scan) - n))
            piece = scan[o:o + n].copy()
        x0[i:i + 1] = gp.moving_state(G @ rv @ synth.exp_so3(3e-3 * g.standard_normal(3)),
                                      np.asarray(gp.G_POS) + G @ (trans + 0.03 * g.standard_normal(3)))
        x0["vel"][i] = g.uniform(-0.5, 0.5, 3)
        P0[i] = _rotated_cov(g, float(g.uniform(0.5, 2.0)))
        if streaming:  # absolute stamps of the hilti kind
            begin = 1.7e9 + 0.1 * i
            piece, offs, times = synth.bucketize(piece, begin_time=begin)
        else:
            begin = 50.0 + 0.37 * i
            offs, times = np.array([0, len(piece)], np.uint32), np.array([begin])
        clk[i]["last_predict_time"] = begin - 0.001 * (1 + i % 5)
        clk[i]["last_update_time"] = begin - 0.0015 * (1 + i % 7)
        bo.extend((offs[1:] + bo[-1]).tolist())
        pieces.append(piece)
        bt.extend(times.tolist())
        sbp.append(sbp[-1] + len(times))
    pts = np.concatenate(pieces)
    so = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.uint32)
    return cfg, blob, x0, P0, clk, pts, so, np.array(sbp, np.uint32), np.array(bo, np.uint32), np.array(bt), [len(p) for p in pieces]


@pytest.mark.parametrize("streaming", [False, True])
def test_heterogeneous_batch(streaming):
    cfg, blob, x0, P0, clk, pts, so, sbp, bo, bt, _ = _hetero_batch(streaming)
    B = len(x0)
    nb = np.diff(sbp)
    if streaming:
        assert (nb > 1).sum() > B // 2 and bt.min() > 1.7e9
    assert pts[so[1]:so[2]].tobytes() == pts[so[0]:so[1]].tobytes()
    Q = abi.process_cov_Q(cfg)
    eng = Engine(cfg)
    eng.map_upload(blob)
    out = eng.scan_update(x0, P0, Q, clk, pts, so, bt, scan_bucket_ptr=sbp, bucket_offsets=bo, iters=2)
    # the same points from two priors: the outputs tell them apart
    assert out["x"][0].tobytes() != out["x"][1].tobytes() and out["P"][0].tobytes() != out["P"][1].tobytes()
    some = 0
    for i in range(B):
        p = pts[so[i]:so[i + 1]]
        if streaming:
            ro, xo, Po, clko = _oracle_stream(cfg, blob, p, 1.7e9 + 0.1 * i, x0[i:i + 1], P0[i], clk[i:i + 1], iters=2)
        else:
            ro, xo, Po, clko = _oracle_bucket(cfg, blob, p, x0[i:i + 1], P0[i], clk[i:i + 1], float(bt[i]), iters=2)
        assert int(out["n_eff"][i]) == ro["n_eff"], (i, len(p))
        assert out["clk"][i].tobytes() == clko.tobytes(), i
        if ro["n_eff"] > 0:
            some += 1
            scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, *HETERO_TOLS, f"scan {i} of {len(p)} points")
        err = np.abs(out["world"][so[i]:so[i + 1], :3] - ro["world"][:, :3])
        assert (err <= gp.world_atol(ro["world"])).all(), (i, err.max())
    assert some >= B - 2
    # the batch reversed: the same per-scan outputs, bitwise, permuted
    r = np.arange(B)[::-1]
    pr = [pts[so[i]:so[i + 1]] for i in r]
    sor = np.concatenate([[0], np.cumsum([len(p) for p in pr])]).astype(np.uint32)
    nbr = [nb[i] for i in r]
    sbpr = np.concatenate([[0], np.cumsum(nbr)]).astype(np.uint32)
    bor = np.concatenate([[0], np.cumsum(np.concatenate([np.diff(bo)[sbp[i]:sbp[i + 1]] for i in r]))]).astype(np.uint32)
    btr = np.concatenate([bt[sbp[i]:sbp[i + 1]] for i in r])
    rev = eng.scan_update(x0[r], P0[r], Q, clk[r], np.concatenate(pr), sor, btr, scan_bucket_ptr=sbpr, bucket_offsets=bor, iters=2)
    for j, i in enumerate(r):
        assert rev["x"][j].tobytes() == out["x"][i].tobytes(), i
        assert rev["P"][j].tobytes() == out["P"][i].tobytes(), i
        assert rev["clk"][j].tobytes() == out["clk"][i].tobytes(), i
        assert rev["n_eff"][j] == out["n_eff"][i]
        assert rev["world"][sor[j]:sor[j + 1]].tobytes() == out["world"][so[i]:so[i + 1]].tobytes(), i
    # cut into two shards: bitwise the same
    for rank in range(2):
        s = shard.shard_batch(rank, 2, x0, P0, clk, pts, so, bt, scan_bucket_ptr=sbp, bucket_offsets=bo)
        part = eng.scan_update(s["x"], s["P"], Q, s["clk"], s["pts"], s["scan_offsets"], s["bucket_times"],
                               scan_bucket_ptr=s["scan_bucket_ptr"], bucket_offsets=s["bucket_offsets"], iters=2)
        assert part["x"].tobytes() == out["x"][s["lo"]:s["hi"]].tobytes()
        assert part["P"].tobytes() == out["P"][s["lo"]:s["hi"]].tobytes()
        assert part["clk"].tobytes() == out["clk"][s["lo"]:s["hi"]].tobytes()
        assert np.array_equal(part["n_eff"], out["n_eff"][s["lo"]:s["hi"]])


# ---- 5. far from the origin ----------------------------------------------------------------------------------------------------

def test_far_from_origin_paths():
    cfg, blob, pts, x0, P0 = _scene_for_rows(gp.FAR_POS, stream=9700)
    _, roots, nodes, _, _ = abi.parse_map_blob(blob)
    assert (roots["key"][:, 0] > 3000).all() and (roots["key"][:, 1] < -5000).all()
    eng = Engine(cfg)
    eng.map_upload(blob)
    ro = _rows_match(eng, cfg, blob, pts, x0, P0)
    # rows that came from the neighbour voxel (the reference's voxel-unit / metre comparison, KILO.cc:158-172): the home
    # root holds a plane whose normal is not the row's
    node_of = {tuple(k): int(n) for k, n in zip(roots["key"].tolist(), roots["node"])}
    took = 0
    for i in np.flatnonzero(ro["ok"]):
        nd = node_of.get(tuple(ro["key"][i].tolist()))
        if nd is not None and nodes["flags"][nd] & abi.NODE_IS_PLANE:
            if np.abs(np.abs(np.dot(nodes["normal"][nd], ro["h"][i, 3:])) - 1.0) > 1e-9:
                took += 1
    print(f"far scene: {int(ro['ok'].sum())} rows, {took} from the neighbour voxel")
    assert took > 0
    clk0 = np.zeros(1, abi.CLOCK_DTYPE); clk0["last_predict_time"] = 99.99; clk0["last_update_time"] = 99.985
    rb, xo, Po, _ = _oracle_bucket(cfg, blob, pts, x0, P0, clk0, 100.0, iters=2)
    Q = abi.process_cov_Q(cfg)
    for fused in (1, 0):
        eng.set_param("fused", fused)
        out = eng.scan_update(x0, P0, Q, clk0, pts, [0, len(pts)], [100.0], iters=2)
        assert int(out["n_eff"][0]) == rb["n_eff"]
        scenes.check_filter(out["x"], out["P"][0], xo, Po, STATE_TOL, COV_TOL, f"fused {fused}")
        err = np.abs(out["world"][:, :3] - rb["world"][:, :3])
        assert (err <= gp.world_atol(rb["world"])).all(), err.max()
    # the batched path: the far scan next to a copy of it at another prior
    x2 = np.concatenate([x0, gp.prior_at(G, gp.FAR_POS, synth.rng(9701))])
    P2 = np.stack([P0, gp.dense_cov(synth.rng(9702))])
    clk2 = np.concatenate([clk0, clk0])
    out = eng.scan_update(x2, P2, Q, clk2, np.concatenate([pts, pts]), [0, len(pts), 2 * len(pts)], [100.0, 100.0], iters=2)
    for i in range(2):
        rb, xo, Po, _ = _oracle_bucket(cfg, blob, pts, x2[i:i + 1], P2[i], clk0, 100.0, iters=2)
        assert int(out["n_eff"][i]) == rb["n_eff"] > 0
        scenes.check_filter(out["x"][i:i + 1], out["P"][i], xo, Po, STATE_TOL, COV_TOL, f"batched scan {i}")
