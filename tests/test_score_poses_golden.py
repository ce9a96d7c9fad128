"""lk_score_poses without a device: tests/golden/ref_score_poses.npz (made by tests/golden/make_ref_score_golden.py from
the reference's own KILO::predictUpdatePoint) against the CPU oracle's rows at every pose, the record layout of the header
against its Python mirror, and the facade's scorePoses member type-checked against the stand-in Eigen of
tests/test_facade_compiles.py. tests/test_gpu_score_poses.py holds the device to the same fixture."""
import os
import re
import subprocess
import tempfile

import numpy as np

import lko
import score_cases as sk
from legkilo_b200 import HEADER_PATH, abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the oracle against the sums stored in the fixture: the same code on the same inputs, so bitwise (any value would do)
ORACLE_TOL = 0.0


def _oracle_record(d, i):
    o = lko.Oracle(abi.CONFIGS["leg_fusion"])
    o.map_import(d["blob"])
    t = float(d["t"])
    clk = np.zeros(1, abi.CLOCK_DTYPE); clk["last_predict_time"] = t; clk["last_update_time"] = t
    o.set_filter(sk.pose_state(d["rot"][i], d["pos"][i]), sk.pose_cov(d["rot_cov"], d["pos_cov"]),
                 abi.process_cov_Q(abi.CONFIGS["leg_fusion"]), clk)
    o.set_options(gain_mode=lko.GAIN_INFORMATION, iters=1, update_map=False)
    r = o.predict_update_point(t, d["pts"], debug=True)
    return sk.row_record(r["ok"], r["h"], r["z"], r["R"])


def test_fixture_counts_match_oracle_rows():
    d = sk.load_fixture()
    assert len(d["counts"]) == 32 and os.path.getsize(sk.GOLD) < 300 * 1024
    # exact, near, far and boundary poses: the far ones lose most of the scan, each boundary pair differs in its count
    assert d["counts"][0] > 0.9 * len(d["pts"]) and (d["counts"][9:18] < 0.5 * d["counts"][0]).all()
    assert all(d["counts"][18 + 2 * k] != d["counts"][19 + 2 * k] for k in range(7))
    assert np.abs(d["pos"][18::2] - d["pos"][19::2]).max() < 1e-6
    for i in range(32):
        rec, scale = _oracle_record(d, i)
        assert int(rec[abi.SCORE_COUNT]) == int(d["counts"][i]), i
        assert sk.record_err(rec, d["oracle_record"][i], scale) <= ORACLE_TOL, i
        assert (scale == d["oracle_scale"][i]).all()


def test_record_layout_mirrors_header():
    src = open(HEADER_PATH).read()
    defs = dict(re.findall(r"#define (LK_SCORE_[A-Z0-9_]+) (\d+)", src))
    assert {k: int(v) for k, v in defs.items()} == {
        "LK_SCORE_A": abi.SCORE_A, "LK_SCORE_B": abi.SCORE_B, "LK_SCORE_SUM_R": abi.SCORE_SUM_R,
        "LK_SCORE_COUNT": abi.SCORE_COUNT, "LK_SCORE_SUM_Z2R": abi.SCORE_SUM_Z2R, "LK_SCORE_STRIDE": abi.SCORE_STRIDE}


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
    const std::vector<double> rec = core.scorePoses(xyzw, offsets, pose_set, rot, pos, Cr, Cp);
    return rec[LK_SCORE_STRIDE + LK_SCORE_COUNT] > 0.0 ? 1 : 0;
}
'''


def test_facade_score_poses_type_checks_against_stub_eigen():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "facade_score_poses.cpp")
        with open(src, "w") as f:
            f.write(FACADE_DRIVER)
        cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"),
               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "leg-kilo_b200", "host"), src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
