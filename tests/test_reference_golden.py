"""Golden vectors made by the REFERENCE ITSELF (tests/golden/make_ref_golden.py: the reference's own eskf.cc /
voxel_map.cc / KILO.cc compiled from /root/reference into oracle/_ref, third-party headers stood in by oracle/ref/shim).
They travel to boxes that have no /root/reference: the CPU oracle is checked against them under -m "not gpu", the CUDA
path — through the C ABI, map built on the device — under -m gpu.

The reference forms the literal n x n gain (eskf.cc:100-107); the CUDA path and the oracle's GAIN_INFORMATION mode form
the algebraically equal 6 x 6 information form, so state / covariance agree to the conditioning of that identity
(1e-7 of the update step here), not to the last bit; success counts, world-cloud intensities, clocks and the map's
structure (every node's flags / point counts) are exact."""
import os

import numpy as np
import pytest

import lko
import mapcmp
import scenes
from legkilo_b200 import abi, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    d = dict(np.load(os.path.join(GOLD, name)))
    for k in ("x0", "x"):
        d[k] = d[k].view(abi.STATE_DTYPE)
    for k in ("clk0", "clk"):
        d[k] = d[k].view(abi.CLOCK_DTYPE)
    return d


# (state_err, cov_err) tolerances (tests/scenes.py) against the fixtures, each at most 100x the worst value measured over
# its tests: the oracle on one bucket in either gain (4.4e-16 sd, 2.2e-16), the oracle on a streaming frame (2.8e-15 sd,
# 4.0e-16), and the device on one bucket / one streaming frame
ORACLE_BUCKET_TOLS = (4e-14, 2e-14)
STREAM_TOLS = (2e-13, 3e-14)
# (on an H100 80GB HBM3: 7.9e-15 sd, 6.5e-16 and 5.4e-13 sd, 2.0e-15)
GPU_BUCKET_TOLS = (7e-13, 6e-14)
GPU_STREAM_TOLS = (5e-11, 1.9e-13)


def _check(d, x, P, clk, world, n_eff, blob, tols, center_atol):
    assert int(n_eff) == int(d["n_eff"]) > 0
    scenes.check_filter(x, P, d["x"], d["P"], *tols)
    assert np.asarray(clk).tobytes() == d["clk"].tobytes()
    np.testing.assert_allclose(world[:, :3], d["world"][:, :3], rtol=0, atol=5e-6)
    np.testing.assert_array_equal(world[:, 3], d["world"][:, 3])
    st = mapcmp.compare_digest(d["map1"], blob, rtol=1e-5, center_atol=center_atol)
    assert st["planes"] > 100


# ---- CPU: oracle against the reference-made fixtures -------------------------------------------------------------------

@pytest.mark.parametrize("cfg_name", ["leg_fusion", "hilti"])
@pytest.mark.parametrize("gain", [lko.GAIN_LITERAL, lko.GAIN_INFORMATION])
def test_oracle_bucket_matches_reference_golden(cfg_name, gain):
    d = _load(f"ref_bucket_{cfg_name}.npz")
    cfg = abi.CONFIGS[cfg_name]
    o = lko.Oracle(cfg)
    o.build_voxel_map(d["pw"], d["pb"])
    mapcmp.compare_digest(d["map0"], o.map_export(), rtol=1e-7, center_atol=1e-12)
    o.set_options(gain_mode=gain, iters=1, update_map=True)
    o.set_filter(d["x0"], abi.init_cov(1), abi.process_cov_Q(cfg), d["clk0"])
    r = o.predict_update_point(float(d["t"]), d["pts"])
    x, P, _, clk = o.get_filter()
    _check(d, x, P, clk, r["world"], r["n_eff"], o.map_export(), ORACLE_BUCKET_TOLS, 1e-9)


@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_oracle_stream_matches_reference_golden(kind):
    d = _load(f"ref_stream_{kind}.npz")
    cfg = abi.CONFIGS["leg_fusion"]
    meas = d["meas"].view(abi.IMU_DTYPE if kind == "imu" else abi.KINIMU_DTYPE)
    o = lko.Oracle(cfg)
    o.build_voxel_map(d["pw"], d["pb"])
    mapcmp.compare_digest(d["map0"], o.map_export(), rtol=1e-7, center_atol=1e-12)
    o.set_options(gain_mode=lko.GAIN_LITERAL, iters=1, update_map=True, imu_mode_only=(kind == "imu"), gravity=9.81, acc_norm=9.79)
    o.set_filter(d["x0"], abi.init_cov(1), abi.process_cov_Q(cfg), d["clk0"])
    r = o.process_scan(float(d["begin"]), d["pts"], **{kind: meas})
    x, P, _, clk = o.get_filter()
    _check(d, x, P, clk, r["world"], r["n_eff"], o.map_export(), STREAM_TOLS, 1e-9)


# ---- GPU: the CUDA path, through the C ABI, against the same fixtures ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", ["leg_fusion", "hilti"])
@pytest.mark.parametrize("fused", [1, 0])
def test_gpu_bucket_matches_reference_golden(cfg_name, fused):
    from legkilo_b200 import Engine
    d = _load(f"ref_bucket_{cfg_name}.npz")
    cfg = abi.CONFIGS[cfg_name]
    eng = Engine(cfg)
    eng.set_param("fused", fused)
    eng.map_build(d["pw"], d["pb"])  # VoxelMapManager::BuildVoxelMap on the device
    mapcmp.compare_digest(d["map0"], eng.map_download(), rtol=1e-6, center_atol=1e-10)
    n = len(d["pts"])
    out = eng.scan_update(d["x0"], abi.init_cov(1), abi.process_cov_Q(cfg), d["clk0"], d["pts"], [0, n], [float(d["t"])], iters=1,
                          update_map=True)
    _check(d, out["x"], out["P"][0], out["clk"], out["world"], out["n_eff"][0], eng.map_download(), GPU_BUCKET_TOLS, 1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["imu", "kin"])
@pytest.mark.parametrize("insert", ["per-bucket", "in-kernel"])
def test_gpu_stream_matches_reference_golden(kind, insert):
    from legkilo_b200 import Engine
    d = _load(f"ref_stream_{kind}.npz")
    cfg = abi.CONFIGS["leg_fusion"]
    meas = d["meas"].view(abi.IMU_DTYPE if kind == "imu" else abi.KINIMU_DTYPE)
    eng = Engine(cfg)
    eng.set_param("fused_insert", 1 if insert == "in-kernel" else 0)
    eng.map_build(d["pw"], d["pb"])
    pts, offs, times = synth.bucketize(d["pts"], begin_time=float(d["begin"]))
    assert pts.tobytes() == d["pts"].tobytes()  # already in the reference's sorted order
    out = eng.process_scan(d["x0"], abi.init_cov(1), abi.process_cov_Q(cfg), d["clk0"], pts, offs, times, imu=meas if kind == "imu" else None,
                           kin=meas if kind == "kin" else None, gravity=9.81, acc_norm=9.79, iters=1, update_map=True)
    _check(d, out["x"], out["P"], out["clk"], out["world"], out["n_eff"], eng.map_download(), GPU_STREAM_TOLS, 1e-8)
