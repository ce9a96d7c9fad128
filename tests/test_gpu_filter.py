"""SURVEY §8f rank 1 on the device: ESKF::updateByPoints from explicit rows, ESKF::predict on a batch of filters,
predictUpdateImu / predictUpdateKinImu, and the full KILO::process bucket loop with the inertial / kinematic queue
interleaved. Every filter is compared with the oracle in its own units (scenes.state_err / scenes.cov_err)."""
import functools

import numpy as np
import pytest

import general_prior as gp
import lko
import scenes
import test_gpu_parity as tp
from legkilo_b200 import Engine, abi, synth

pytestmark = pytest.mark.gpu
# (state_err, cov_err) tolerances (tests/scenes.py), each 100x the worst measured on an H100 80GB HBM3: explicit rows
# and inertial / kinematic samples 8.8e-14 sd / 1.3e-14; predict 2.8e-14 sd / 1.8e-16; a scan with its queue and a static
# map 6.6e-13 sd / 5.3e-15, with UpdateVoxelMap 1.2e-8 sd / 8.8e-12
STATE_TOL = 8e-12
COV_TOL = 1.3e-12
PREDICT_STATE_TOL = 2.7e-12
PREDICT_COV_TOL = 1.7e-14
QUEUE_TOLS = {False: (6e-11, 5e-13), True: (1.1e-6, 8e-10)}  # by update_map
CFG = abi.CONFIGS["leg_fusion"]


def _filter(seed):
    g = synth.rng(seed)
    A = g.standard_normal((30, 30)) * 1e-3
    P = A @ A.T + 1e-6 * np.eye(30)
    x = tp._moving_state()
    x["rot"][0] = lko.exp3(g.normal(size=3) * 0.1).ravel()
    return x, P


@pytest.mark.parametrize("n", [1, 2, 40, 3000])
def test_update_by_points_rows(n):
    g = synth.rng(300 + n)
    x0, P0 = _filter(n)
    h = g.standard_normal((n, 6)); z = g.standard_normal(n) * 1e-2; r = g.uniform(1e-3, 1e-2, n)
    o = lko.Oracle(CFG); o.set_filter(x0, P0.ravel(), None, None)
    o.update_by_points(h, z, r, gain_mode=lko.GAIN_LITERAL if n <= 40 else lko.GAIN_INFORMATION)
    xo, Po, _, _ = o.get_filter()
    xg, Pg = Engine(CFG).update_by_points(x0, P0, h, z, r)
    scenes.check_filter(xg, Pg, xo, Po, STATE_TOL, COV_TOL)


PREDICT_DTS = (0.0, 1e-4, 0.0123, 0.1, -0.005, 0.5)


def test_predict_kernel():
    """Six filters in one lk_predict call, each at its own general prior (attitude anywhere on SO(3), moving, dense P) and
    its own dt, zero and negative ones included, in all four (prop_state, prop_cov) modes. Each equals the oracle, and
    bitwise the same filter predicted alone."""
    g = synth.rng(77)
    B = len(PREDICT_DTS)
    x0 = np.concatenate([gp.prior_at(gp.so3_uniform(g), g.uniform(-50.0, 50.0, 3), g) for _ in range(B)])
    x0["vel"] = g.uniform(-1.0, 1.0, (B, 3))
    P0 = np.stack([gp.dense_cov(g, scale=float(g.uniform(0.5, 2.0))) for _ in range(B)])
    Q = abi.process_cov_Q(CFG)
    eng = Engine(CFG)
    for ps, pc in ((True, True), (True, False), (False, True), (False, False)):
        xg, Pg = eng.predict(x0, P0, Q, PREDICT_DTS, ps, pc)
        for i, dt in enumerate(PREDICT_DTS):
            what = f"prop_state {ps} prop_cov {pc} dt {dt}"
            o = lko.Oracle(CFG); o.set_filter(x0[i:i + 1], P0[i], Q, None); o.predict(dt, ps, pc)
            xo, Po, _, _ = o.get_filter()
            scenes.check_filter(xg[i:i + 1], Pg[i], xo, Po, PREDICT_STATE_TOL, PREDICT_COV_TOL, what)
            xa, Pa = eng.predict(x0[i:i + 1], P0[i:i + 1], Q, [dt], ps, pc)
            assert xa.tobytes() == xg[i:i + 1].tobytes() and Pa.tobytes() == Pg[i:i + 1].tobytes(), what
            if not ps:
                assert xg[i:i + 1].tobytes() == x0[i:i + 1].tobytes(), what
            if not pc:
                assert Pg[i].tobytes() == P0[i].tobytes(), what


def _contact_subsets(kin):
    """Cycles the kinematic samples through all 16 contact subsets (m = 6 ... 18); some in-contact legs read 2 or -1."""
    kin = kin.copy()
    for i in range(len(kin)):
        bits = np.array([(i % 16) >> leg & 1 for leg in range(4)], np.int32)
        if i % 5 == 1:
            bits *= 2
        elif i % 5 == 3:
            bits *= -1
        kin["contact"][i] = bits
    return kin


def _obs_stream(kind, t_update, t_predict):
    """A queue whose first sample sits at last_update_time (dtc = 0) and behind last_predict_time (dt < 0), with one
    stamp repeated (dt = 0) and one sample that steps back in time."""
    meas = synth.imu_stream(t_predict, t_predict + 0.05) if kind == "imu" else _contact_subsets(synth.kinimu_stream(t_predict, t_predict + 0.05))
    meas = np.concatenate([meas[:1], meas])
    meas["stamp"][0] = t_update
    meas["stamp"][7] = meas["stamp"][6]
    meas["stamp"][12] = meas["stamp"][11] - 0.001
    return meas


@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_inertial_and_kinematic_observations(kind):
    g = synth.rng(9)
    x0 = gp.prior_at(gp.so3_uniform(g), (12.0, -7.5, 0.4), g)
    P0 = gp.dense_cov(g)
    Q = abi.process_cov_Q(CFG)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 3.0; clk["last_update_time"] = 2.995
    meas = _obs_stream(kind, 2.995, 3.0)
    if kind == "kin":
        nc = (meas["contact"] != 0).sum(axis=1)
        assert set(nc.tolist()) == {0, 1, 2, 3, 4} and (meas["contact"] == 2).any() and (meas["contact"] == -1).any()
    o = lko.Oracle(CFG); o.set_filter(x0, P0, Q, clk); o.set_options(imu_mode_only=(kind == "imu"), gravity=9.81, acc_norm=9.79)
    (o.obs_imu if kind == "imu" else o.obs_kinimu)(meas)
    xo, Po, _, co = o.get_filter()
    eng = Engine(CFG)
    xg, Pg, cg = (eng.obs_imu if kind == "imu" else eng.obs_kinimu)(x0, P0, Q, clk, meas, gravity=9.81, acc_norm=9.79)
    scenes.check_filter(xg, Pg, xo, Po, STATE_TOL, COV_TOL)
    assert cg.tobytes() == co.tobytes()


@functools.lru_cache(maxsize=None)
def _queue_scene():
    cfg, blob, scans = scenes.box_scene(batch=1, streaming=True, stream0=1100)
    pts, offs, times = synth.bucketize(scans[0], begin_time=20.0)
    return cfg, blob, pts, offs, times


def _queue(kind, shape, times):
    """The inertial / kinematic queue of one scan, shaped as `shape` names. Returns it and the samples the scan consumes
    (those stamped before the last bucket)."""
    mk = synth.imu_stream if kind == "imu" else synth.kinimu_stream
    meas = mk(19.996, 20.12)
    if shape == "at-bucket-times":  # a sample exactly at an inner bucket's time and one exactly at the last bucket's
        for t in (times[len(times) // 2], times[-1]):
            meas["stamp"][np.searchsorted(meas["stamp"], t)] = t
    elif shape == "duplicates":  # three equal stamps between two buckets
        j = np.searchsorted(meas["stamp"], times[10])
        meas = np.concatenate([meas[:j], meas[j:j + 1], meas[j:j + 1], meas[j:]])
        assert times[10] < meas["stamp"][j] == meas["stamp"][j + 2] < times[11]
    elif shape == "before":
        meas = mk(19.9951, 19.9999, rate_hz=2000.0)
    elif shape == "after":
        meas = mk(float(times[-1]) + 1e-4, float(times[-1]) + 0.03)
    elif shape == "empty":
        meas = meas[:0]
    elif shape == "contact-subsets":
        meas = _contact_subsets(meas)
    return meas, int((meas["stamp"] < times[-1]).sum())


PATHS = {"fused": (False, 0), "per-bucket": (True, 0), "in-kernel": (True, 1)}
SHAPES = ["stream", "at-bucket-times", "duplicates", "before", "after", "empty"]


@pytest.mark.parametrize("kind,shape", [(k, s) for k in ("imu", "kin") for s in SHAPES] + [("kin", "contact-subsets")])
@pytest.mark.parametrize("path", list(PATHS))
def test_process_scan_with_interleaved_queue(path, kind, shape):
    """KILO::process's second lambda: ~50 buckets, every sample with stamp < bucket time applied first
    (KILO.cc:379-390). "fused" runs the fused persistent kernel (fused_drain_queue) with a static map, "per-bucket" the
    per-bucket kernels (k_obs_predict_prepare) with UpdateVoxelMap, "in-kernel" the persistent kernel with UpdateVoxelMap
    inside (queue drain, predict, update and insert of all buckets in ONE launch). The queue shapes put samples exactly
    at bucket times, repeat stamps, lie wholly before the first bucket or after the last, or are empty."""
    update_map, fused_insert = PATHS[path]
    cfg, blob, pts, offs, times = _queue_scene()
    meas, n_before_last = _queue(kind, shape, times)
    x0 = tp._moving_state(); P0 = abi.init_cov(1)
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = 19.995; clk["last_update_time"] = 19.995
    Q = abi.process_cov_Q(cfg)
    q = dict(imu=meas if kind == "imu" else None, kin=meas if kind == "kin" else None)
    o = lko.Oracle(cfg); o.map_import(blob); o.set_filter(x0, P0, Q, clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, update_map=update_map, imu_mode_only=(kind == "imu"), gravity=9.81, acc_norm=9.79)
    ro = o.process_scan(20.0, pts, **q)
    xo, Po, _, co = o.get_filter()
    eng = Engine(cfg); eng.map_upload(blob)
    eng.set_param("fused_insert", fused_insert)
    out = eng.process_scan(x0, P0, Q, clk, pts, offs, times, **q, gravity=9.81, acc_norm=9.79, update_map=update_map)
    assert out["n_consumed"] == ro["n_consumed"] == n_before_last and out["n_eff"] == ro["n_eff"] > 0
    if shape in ("stream", "duplicates", "contact-subsets"):
        assert n_before_last > 30
    elif shape == "at-bucket-times":  # the sample at the last bucket's time stays queued
        assert meas["stamp"][n_before_last] == times[-1]
    elif shape == "before":
        assert n_before_last == len(meas) > 5
    scenes.check_filter(out["x"], out["P"], xo, Po, *QUEUE_TOLS[update_map])
    assert out["clk"].tobytes() == co.tobytes()
    np.testing.assert_allclose(out["world"][:, :3], ro["world"][:, :3], rtol=0, atol=1e-5)
    if shape == "after":  # nothing is drained: the call equals the same call without a queue, bit for bit
        eng2 = Engine(cfg); eng2.map_upload(blob)
        eng2.set_param("fused_insert", fused_insert)
        bare = eng2.process_scan(x0, P0, Q, clk, pts, offs, times, gravity=9.81, acc_norm=9.79, update_map=update_map)
        assert out["n_consumed"] == 0 and bare["n_consumed"] == 0
        for k in ("x", "P", "clk"):
            assert np.asarray(out[k]).tobytes() == np.asarray(bare[k]).tobytes(), k
