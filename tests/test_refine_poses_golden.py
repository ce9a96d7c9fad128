"""lk_refine_poses without a device: the reference's chains of tests/golden/ref_refine_poses.npz (made by
tests/golden/make_ref_refine_golden.py from KILO::predictUpdatePoint with P held) against the step restated in numpy
(refine_cases.step_delta) on the CPU oracle's rows at each pose of the chain, and the facade's refinePoses member
type-checked against the stand-in Eigen of tests/test_facade_compiles.py. tests/test_gpu_refine_poses.py holds the device
to the same fixture."""
import os
import subprocess
import tempfile

import numpy as np

import lko
import refine_cases as rk
import score_cases as sk
from legkilo_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the information-form step on the oracle's float64 rows against the reference's literal gain, per step (m / rad)
STEP_TOL = 1e-11


def _oracle_rows(d, R, p):
    o = lko.Oracle(abi.CONFIGS["leg_fusion"])
    o.map_import(d["blob"])
    t = float(d["t"])
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = t; clk["last_update_time"] = t
    o.set_filter(sk.pose_state(R, p), sk.pose_cov(d["rot_cov"], d["pos_cov"]), abi.process_cov_Q(abi.CONFIGS["leg_fusion"]),
                 clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    r = o.predict_update_point(t, d["pts"], debug=True)
    m = np.asarray(r["ok"]).astype(bool)
    return np.asarray(r["h"])[m], np.asarray(r["z"])[m], np.asarray(r["R"])[m]


def test_fixture_chain_is_the_restated_step():
    d, g = sk.load_fixture(), rk.load_fixture()
    assert os.path.getsize(rk.GOLD) < 32 * 1024
    assert g["rot"].shape == (len(rk.POSES), rk.K + 1, 3, 3) and (g["poses"] == rk.POSES).all()
    worst, worst_gain = 0.0, 0.0
    for j, i in enumerate(rk.POSES):
        assert np.array_equal(g["rot"][j, 0], d["rot"][i]) and np.array_equal(g["pos"][j, 0], d["pos"][i])
        for k in range(rk.K):
            R, p = g["rot"][j, k], g["pos"][j, k]
            h, z, r = _oracle_rows(d, R, p)
            assert len(z) == g["counts"][j, k], (i, k)
            rec, _ = sk.row_record(np.ones(len(z)), h, z, r)
            delta = rk.step_delta(rec, d["rot_cov"], d["pos_cov"])
            Rn, pn = rk.boxplus(R, p, delta)
            worst = max(worst, np.abs(Rn - g["rot"][j, k + 1]).max(), np.abs(pn - g["pos"][j, k + 1]).max())
            worst_gain = max(worst_gain, np.abs(delta - rk.gain_delta(h, z, r, d["rot_cov"], d["pos_cov"])).max())
    print(f"[refine] restated step against the reference's chain: {worst:.3g}; information form against the literal gain "
          f"{worst_gain:.3g}")
    assert worst <= STEP_TOL and worst_gain <= STEP_TOL
    # the chains move: the near and far poses approach the exact one
    assert np.abs(g["pos"][1:, -1] - g["pos"][1:, 0]).max() > 1e-3


FACADE_DRIVER = r'''
#include <vector>
#include "legkilo_facade.hpp"
using namespace legkilo::b200;
struct EskfConfig { double v[14]; };
struct VoxelMapConfig {
    double max_voxel_size_, planner_threshold_, beam_err_, dept_err_, sigma_num_;
    int max_layer_, max_points_num_;
    std::vector<int> layer_init_num_;
};
int main() {
    EskfConfig ec{}; VoxelMapConfig mc{}; mc.layer_init_num_ = {5, 5, 5, 5, 5};
    Mat3D Re, Cr, Cp; Vec3D te;
    Core core(ec, mc, Re, te, 0);
    std::vector<float> xyzw(8);
    std::vector<uint32_t> offsets = {0, 2}, pose_set = {0, 0};
    std::vector<Mat3D> rot(2);
    std::vector<Vec3D> pos(2);
    const std::vector<double> rec = core.refinePoses(xyzw, offsets, pose_set, rot, pos, Cr, Cp, 10);
    return rec[LK_SCORE_STRIDE + LK_SCORE_COUNT] > 0.0 ? 1 : 0;
}
'''


def test_facade_refine_poses_type_checks_against_stub_eigen():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "facade_refine_poses.cpp")
        with open(src, "w") as f:
            f.write(FACADE_DRIVER)
        cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"),
               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "leg-kilo_b200", "host"), src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
