"""lk_first_frame: the first frame of KILO::process (KILO.cc:331-353) in one device call, against the reference-made fixtures
(tests/golden/ref_first_frame_*.npz), against the manual path it replaces (host StateInitial, host cloudLidarToWorld,
lk_map_build), and at its edges."""
import numpy as np
import pytest

import mapcmp
import scenes
from first_frame_cases import canonical_map, first_frame_numpy, lidar_to_world_numpy, load_first_frame, os64_raw_scan, sha256
from legkilo_b200 import abi, synth

pytestmark = pytest.mark.gpu

CFG = abi.CONFIGS["leg_fusion"]
# (state_err, cov_err) bounds of the device against the reference after streaming frames 1 and 2, which start from the
# device's own first frame: GPU_STREAM_TOLS of tests/test_reference_golden.py, the bounds of one streaming frame
# (on an H100 80GB HBM3: at most 1.4e-12 sd and 5.7e-14 over both frames and both modes)
FRAME_TOLS = (5e-11, 1.9e-13)


def _engine():
    from legkilo_b200 import Engine
    return Engine(CFG)


def _queue(d, kind, f):
    return {kind: d[f"meas{f}"]}


def _manual_map(raw, pos=(0.0, 0.0, 0.0)):
    """The map of INTEGRATION §3 before lk_first_frame: cloudLidarToWorld on the host at rot = I, then lk_map_build with
    StateInitial's P = 1e-6 I blocks. Canonical bytes (canonical_map)."""
    eng = _engine()
    world = lidar_to_world_numpy(raw, CFG, pos=pos)
    eng.map_build(world[:, :3], raw[:, :3], R=np.eye(3), rot_cov=1e-6 * np.eye(3), pos_cov=1e-6 * np.eye(3))
    return canonical_map(eng.map_download())


def _check_state_initial(out, x_prior, meas):
    grav, bw, acc_norm = first_frame_numpy(meas, 9.81)
    x = out["x"]
    np.testing.assert_allclose(x["grav"][0], grav, rtol=0, atol=1e-12)
    np.testing.assert_allclose(x["bw"][0], bw, rtol=0, atol=1e-14)
    assert abs(out["acc_norm"] - acc_norm) < 1e-12
    assert x["rot"].tobytes() == np.eye(3).tobytes()
    for f in abi.STATE_DTYPE.names:
        if f not in ("grav", "bw", "rot"):
            assert x[f].tobytes() == x_prior[f].tobytes(), f
    assert out["P"].tobytes() == abi.init_cov(1).ravel().tobytes()


@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_first_frame_matches_reference_golden(kind):
    d = load_first_frame(kind)
    eng = _engine()
    out = eng.first_frame(abi.default_states(1), d["raw0"], float(d["end0"]), gravity=9.81, **_queue(d, kind, 0))
    x = out["x"]
    np.testing.assert_allclose(x["grav"][0], d["x0"]["grav"][0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(x["bw"][0], d["x0"]["bw"][0], rtol=0, atol=1e-14)
    assert abs(out["acc_norm"] - float(d["acc_norm"])) < 1e-12
    for f in abi.STATE_DTYPE.names:
        if f not in ("grav", "bw"):
            assert x[f].tobytes() == d["x0"][f].tobytes(), f
    assert out["P"].tobytes() == d["P0"].tobytes()
    assert out["clk"].tobytes() == d["clk0"].tobytes()
    assert sha256(out["world"]) == str(d["world0_sha256"])
    st = mapcmp.compare_digest(d["map0_digest"], eng.map_download(), rtol=1e-6, center_atol=1e-10)
    assert st["planes"] > 100
    # frames 1-2 stream on from the device's own first frame, acc_norm taken from the call
    Q = abi.process_cov_Q(CFG)
    xs, P, clk = out["x"], out["P"], out["clk"]
    for f in (1, 2):
        pts, offs, times = synth.bucketize(d[f"body{f}"], begin_time=float(d[f"begin{f}"]))
        assert pts.tobytes() == d[f"body{f}"].tobytes()  # already in the reference's sorted order
        r = eng.process_scan(xs, P, Q, clk, pts, offs, times, gravity=9.81, acc_norm=out["acc_norm"], iters=1, update_map=True,
                             **_queue(d, kind, f))
        xs, P, clk = r["x"], r["P"], r["clk"]
        assert r["n_eff"] == int(d[f"n_eff{f}"]) > 0
        scenes.check_filter(xs, P, d[f"x{f}"], d[f"P{f}"], *FRAME_TOLS, what=f"frame {f}")
        assert clk.tobytes() == d[f"clk{f}"].tobytes()
        np.testing.assert_allclose(r["world"][:, :3], d[f"world{f}"][:, :3], rtol=0, atol=5e-6)
        np.testing.assert_array_equal(r["world"][:, 3], d[f"world{f}"][:, 3])


@pytest.mark.parametrize("cloud", ["fixture", "os64"])
def test_first_frame_map_equals_the_manual_path(cloud):
    if cloud == "fixture":
        d = load_first_frame("imu")
        raw, meas = d["raw0"], d["meas0"]
    else:
        raw, meas = os64_raw_scan(CFG), synth.imu_stream(9.9, 10.0)
    x0 = abi.default_states(1)
    eng = _engine()
    out = eng.first_frame(x0, raw, 10.0, imu=meas)
    assert out["world"].tobytes() == lidar_to_world_numpy(raw, CFG).tobytes()
    assert canonical_map(eng.map_download()) == _manual_map(raw)
    assert eng.map_stats()["roots"] > 100


def test_prior_fields_pass_through():
    d = load_first_frame("kin")
    x0 = abi.default_states(1)
    x0["rot"][0] = synth.exp_so3([0.1, -0.2, 0.3]).ravel()
    x0["pos"][0] = (3.25, -1.5, 0.75)
    x0["vel"][0] = (0.4, -0.2, 0.05)
    x0["ba"][0] = (0.01, -0.02, 0.03)
    x0["bw"][0] = (1e-3, 2e-3, -1e-3)
    x0["grav"][0] = (0.1, 0.2, -9.7)
    x0["imu_a"][0] = (0.3, 0.1, 9.7)
    x0["imu_w"][0] = (0.02, -0.03, 0.15)
    x0["bv"][0] = (-0.01, 0.02, 0.0)
    x0["contact"][0] = (0.5, -0.25, -0.4)
    eng = _engine()
    out = eng.first_frame(x0, d["raw0"], 50.0, kin=d["meas0"])
    _check_state_initial(out, x0, d["meas0"])
    assert out["world"].tobytes() == lidar_to_world_numpy(d["raw0"], CFG, pos=x0["pos"][0]).tobytes()
    assert canonical_map(eng.map_download()) == _manual_map(d["raw0"], pos=x0["pos"][0])


def _raw_call(eng, x, P, clk, acc, pts, n_pts, imu, kin, n_meas, world):
    from legkilo_b200 import _p, lib
    return lib().lk_first_frame(eng.h, _p(x), _p(P), _p(clk), _p(acc), _p(pts), n_pts, 50.0, _p(imu), _p(kin), n_meas, 9.81,
                                _p(world))


def test_not_ready_writes_nothing_and_keeps_the_map():
    d = load_first_frame("imu")
    raw, imu = d["raw0"], d["meas0"]
    kin = load_first_frame("kin")["meas0"]
    eng = _engine()
    eng.map_build(lidar_to_world_numpy(raw, CFG)[:, :3], raw[:, :3])
    stats0, map0 = eng.map_stats(), canonical_map(eng.map_download())
    x_in = abi.default_states(1); x_in["pos"][0] = (1.0, 2.0, 3.0)
    empty_imu = np.zeros(0, abi.IMU_DTYPE)
    cases = [(raw, 0, imu, None, len(imu)),           # empty cloud
             (raw, len(raw), empty_imu, None, 0),     # empty IMU queue
             (raw, len(raw), None, kin[:0], 0),       # empty Kin+IMU queue
             (raw, len(raw), None, None, 0)]          # no queue at all
    for pts, n_pts, q_imu, q_kin, n_meas in cases:
        x = x_in.copy(); P = np.full(900, -7.0); clk = np.full(1, -7.0, dtype=[("a", "f8"), ("b", "f8")])
        acc = np.full(1, -7.0); world = np.full((len(raw), 4), -7.0, np.float32)
        assert _raw_call(eng, x, P, clk, acc, pts, n_pts, q_imu, q_kin, n_meas, world) == -7  # LK_ERR_NOT_READY
        assert x.tobytes() == x_in.tobytes() and (P == -7.0).all() and (acc == -7.0).all() and (world == -7.0).all()
        assert (clk["a"] == -7.0).all() and (clk["b"] == -7.0).all()
        assert eng.map_stats() == stats0
    assert canonical_map(eng.map_download()) == map0


@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_one_sample_queue(kind):
    d = load_first_frame(kind)
    s = d["meas0"][3:4].copy()
    eng = _engine()
    out = eng.first_frame(abi.default_states(1), d["raw0"], 50.0, world=False, **{kind: s})
    a = s["acc"][0]
    np.testing.assert_allclose(out["x"]["grav"][0], -a / np.linalg.norm(a) * 9.81, rtol=0, atol=1e-12)
    assert out["x"]["bw"][0].tobytes() == s["gyr"][0].tobytes()
    assert out["world"] is None


def test_invalid_arguments():
    from legkilo_b200 import LkError
    d = load_first_frame("imu")
    raw, imu = d["raw0"], d["meas0"]
    kin = load_first_frame("kin")["meas0"]
    eng = _engine()
    with pytest.raises(LkError) as e:
        eng.first_frame(abi.default_states(1), raw, 50.0, imu=imu, kin=kin[:len(imu)])
    assert e.value.code == -1
    x = abi.default_states(1); P = np.zeros(900); clk = np.zeros(1, abi.CLOCK_DTYPE); acc = np.zeros(1)
    args = dict(x=x, P=P, clk=clk, acc=acc, pts=raw)
    for k in args:
        a = dict(args, **{k: None})
        assert _raw_call(eng, a["x"], a["P"], a["clk"], a["acc"], a["pts"], len(raw), imu, None, len(imu), None) == -1, k
    assert _raw_call(eng, x, P, clk, acc, raw, len(raw), None, None, len(imu), None) == -1  # n_meas without samples
    from legkilo_b200 import lib
    assert lib().lk_first_frame(None, None, None, None, None, None, 0, 0.0, None, None, 0, 9.81, None) == -1


def test_second_call_replaces_the_map():
    d = load_first_frame("imu")
    eng = _engine()
    eng.first_frame(abi.default_states(1), d["raw0"], 50.0, imu=d["meas0"])
    other = os64_raw_scan(CFG)[::7].copy()
    eng.first_frame(abi.default_states(1), other, 60.0, imu=d["meas0"])
    fresh = _engine()
    fresh.first_frame(abi.default_states(1), other, 60.0, imu=d["meas0"])
    assert canonical_map(eng.map_download()) == canonical_map(fresh.map_download())
    assert eng.map_stats() == fresh.map_stats()
