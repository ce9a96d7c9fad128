"""lk_search_poses without a device: the candidate lattice of tests/search_cases.py against a brute-force loop over the
header's formula, and the facade's searchPoses member type-checked against the stand-in Eigen of
tests/test_facade_compiles.py. tests/test_gpu_search_poses.py holds the device to the composition built on that lattice."""
import os
import subprocess
import tempfile

import numpy as np

import search_cases as xs
from legkilo_b200 import synth

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))


def test_lattice_matches_the_header_formula():
    g = synth.rng(1230)
    att = np.array([synth.exp_so3(g.normal(0.0, 0.3, 3)) for _ in range(3)])
    origin, step, counts = g.normal(0.0, 5.0, 3), np.array([0.1, 0.3, 0.7]), (4, 3, 2)
    rot, pos = xs.lattice(att, origin, step, counts)
    L = 4 * 3 * 2
    assert rot.shape == (3 * L, 3, 3) and pos.shape == (3 * L, 3)
    c = 0
    for a in range(3):
        for iz in range(2):
            for iy in range(3):
                for ix in range(4):
                    assert c // L == a and (c % L) % 4 == ix and ((c % L) // 4) % 3 == iy and (c % L) // 12 == iz
                    assert rot[c].tobytes() == att[a].tobytes()
                    want = [float(origin[j]) + float(i) * float(step[j]) for j, i in enumerate((ix, iy, iz))]
                    assert pos[c].tobytes() == np.array(want).tobytes(), c
                    c += 1
    # a slice is the same candidates
    r2, p2 = xs.lattice(att, origin, step, counts, 17, 30)
    assert r2.tobytes() == rot[17:47].tobytes() and p2.tobytes() == pos[17:47].tobytes()
    r3, p3 = xs.lattice_at(att, origin, step, counts, [71, 0, 5])
    assert r3.tobytes() == rot[[71, 0, 5]].tobytes() and p3.tobytes() == pos[[71, 0, 5]].tobytes()


def test_keys_order_count_then_index():
    k = xs.keys(np.array([3.0, 5.0, 3.0, 0.0, 5.0]), 10)
    assert list((np.sort(k) & np.uint64(0xFFFFFFFF)).astype(int)) == [11, 14, 10, 12, 13]


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
    Mat3D Re, Cr, Cp; Vec3D te, step;
    Core core(ec, mc, Re, te, 0);
    std::vector<float> xyzw(8);
    std::vector<uint32_t> offsets = {0, 2}, att_offsets = {0, 3}, cand;
    std::vector<Mat3D> att(3), rot;
    std::vector<Vec3D> origin(1), pos;
    const uint32_t counts[3] = {21, 21, 1};
    const std::vector<double> rec = core.searchPoses(xyzw, offsets, att_offsets, att, origin, step, counts, Cr, Cp, 10, Cr, Cp,
                                                     8, rot, pos, cand);
    return rec[LK_SCORE_COUNT] > 0.0 && cand[0] == 0u ? 1 : 0;
}
'''


def test_facade_search_poses_type_checks_against_stub_eigen():
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "facade_search_poses.cpp")
        with open(src, "w") as f:
            f.write(FACADE_DRIVER)
        cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"),
               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "leg-kilo_b200", "host"), src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
