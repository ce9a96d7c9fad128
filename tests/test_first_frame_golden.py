"""The first frame of KILO::process (KILO.cc:331-353) as the reference computed it (tests/golden/ref_first_frame_*.npz, made by
tests/golden/make_ref_first_frame_golden.py from the reference's own KILO.cc): the fixtures checked against a numpy
restatement of StateInitial and of cloudLidarToWorld, and the CPU oracle's BuildVoxelMap from the fixture's world cloud
against the reference's map. tests/test_gpu_first_frame.py holds lk_first_frame to the same fixtures. Also type-checks the
facade's firstFrame member against the stand-in Eigen of tests/test_facade_compiles.py."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import lko
import mapcmp
from first_frame_cases import first_frame_numpy, lidar_to_world_numpy, load_first_frame, sha256
from legkilo_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind", ["imu", "kin"])
def test_fixture_matches_numpy_state_initial(kind):
    d = load_first_frame(kind)
    cfg = abi.CONFIGS["leg_fusion"]
    grav, bw, acc_norm = first_frame_numpy(d["meas0"], 9.81)
    x = d["x0"]
    assert abs(float(d["acc_norm"]) - acc_norm) < 1e-12
    np.testing.assert_allclose(x["grav"][0], grav, rtol=0, atol=1e-12)
    np.testing.assert_allclose(x["bw"][0], bw, rtol=0, atol=1e-14)
    # every other field is the fresh node's state; P = 1e-6 I; both clocks at the frame's end
    x_def = abi.default_states(1)
    for f in abi.STATE_DTYPE.names:
        if f not in ("grav", "bw"):
            assert x[f].tobytes() == x_def[f].tobytes(), f
    assert d["P0"].tobytes() == abi.init_cov(1).ravel().tobytes()
    assert float(d["clk0"]["last_predict_time"][0]) == float(d["clk0"]["last_update_time"][0]) == float(d["end0"])
    assert sha256(lidar_to_world_numpy(d["raw0"], cfg)) == str(d["world0_sha256"])


def test_oracle_rebuilds_the_fixture_map_from_the_world_cloud():
    """The world cloud restated above (bitwise the reference's), through the oracle's BuildVoxelMap, against the digest of
    the reference's map at the bounds of the other oracle-vs-reference-fixture map checks (test_reference_golden.py)."""
    d = load_first_frame("imu")
    P = d["P0"].reshape(30, 30)
    world = lidar_to_world_numpy(d["raw0"], abi.CONFIGS["leg_fusion"])
    o = lko.Oracle(abi.CONFIGS["leg_fusion"])
    o.build_voxel_map(world[:, :3], d["raw0"][:, :3], R=np.eye(3), rot_cov=P[:3, :3], pos_cov=P[3:6, 3:6])
    st = mapcmp.compare_digest(d["map0_digest"], o.map_export(), rtol=1e-7, center_atol=1e-12)
    assert st["planes"] > 100
    # the kin fixture's frame 0 built the same map (only grav / bw differ between the modes)
    assert load_first_frame("kin")["map0_digest"].tobytes() == d["map0_digest"].tobytes()


FACADE_DRIVER = r'''
#include <vector>
#include "legkilo_facade.hpp"
using namespace legkilo::b200;
struct State { Mat3D rot_; Vec3D pos_, vel_, ba_, bw_, grav_, imu_a_, imu_w_, bv_, contact_; };
struct EskfConfig { double v[14]; };
struct VoxelMapConfig {
    double max_voxel_size_, planner_threshold_, beam_err_, dept_err_, sigma_num_;
    int max_layer_, max_points_num_;
    std::vector<int> layer_init_num_;
};
int main() {
    EskfConfig ec{}; VoxelMapConfig mc{}; mc.layer_init_num_ = {5, 5, 5, 5, 5};
    Mat3D Re; Vec3D te;
    Core core(ec, mc, Re, te, 0);
    State s; StateCov P; double tp = 0, tu = 0, acc_norm = 0;
    std::vector<float> raw, world;
    std::vector<lk_imu_meas> imu; std::vector<lk_kinimu_meas> kin;
    bool ok = core.firstFrame(s, P, tp, tu, acc_norm, raw, 50.0, imu, kin, 9.81, &world);
    ok = ok && core.firstFrame(s, P, tp, tu, acc_norm, raw, 50.0, imu, kin, 9.81);
    return ok ? 1 : 0;
}
'''


def test_facade_first_frame_type_checks_against_stub_eigen():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "facade_first_frame.cpp")
        with open(src, "w") as f:
            f.write(FACADE_DRIVER)
        cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"),
               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "leg-kilo_b200", "host"), src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
