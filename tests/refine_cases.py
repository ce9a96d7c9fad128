"""lk_refine_poses restated on the host, and its reference fixture (tests/golden/ref_refine_poses.npz, written by
tests/golden/make_ref_refine_golden.py from the scene of tests/golden/ref_score_poses.npz).

One step from a record (include/legkilo_b200.h: LK_SCORE_*) at the current pose, with P66 = blockdiag(sym(rot_cov),
sym(pos_cov)): y = (I + A P66)^-1 b, delta = P66 y (the N == 1 rule scales A and b by sum R / (sum R + 1e-4)), then
State::operator+= (eskf.cc:18-29): R <- R Exp(delta_theta), p <- p + delta_p.

Shared by tests/golden/make_ref_refine_golden.py, tests/test_refine_poses_golden.py (CPU) and
tests/test_gpu_refine_poses.py."""
import os

import numpy as np

import score_cases as sk
from legkilo_b200 import abi, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_refine_poses.npz")
# the poses of ref_score_poses.npz the fixture refines: exact (0), near (1..8), far (9..17)
POSES = np.arange(18)
K = 5  # reference steps per chain


def p66(rot_cov, pos_cov):
    P = np.zeros((6, 6))
    P[:3, :3] = 0.5 * (rot_cov + rot_cov.T)
    P[3:, 3:] = 0.5 * (pos_cov + pos_cov.T)
    return P


def unpack(rec):
    """A (6 x 6), b (6), sum R and count of a record."""
    A = np.zeros((6, 6))
    A[sk.IU] = rec[abi.SCORE_A:abi.SCORE_A + 21]
    A = A + np.triu(A, 1).T
    return A, np.array(rec[abi.SCORE_B:abi.SCORE_B + 6]), rec[abi.SCORE_SUM_R], rec[abi.SCORE_COUNT]


def step_delta(rec, rot_cov, pos_cov):
    """delta (6) of one step from a record; zero when the count is 0."""
    A, b, sum_r, cnt = unpack(rec)
    if cnt < 0.5:
        return np.zeros(6)
    if cnt < 1.5:  # N == 1 adds 1e-4 to S (eskf.cc:100)
        s = sum_r / (sum_r + 1e-4)
        A, b = A * s, b * s
    P = p66(rot_cov, pos_cov)
    y = np.linalg.solve(np.eye(6) + A @ P, b)
    return P @ y


def gain_delta(h, z, r, rot_cov, pos_cov):
    """delta (6) of one step from the rows themselves, by ESKF::updateByPoints' literal gain restricted to the pose:
    K = P66 H^T (H P66 H^T + R)^-1 (1e-4 added to S when there is one row), delta = K z."""
    if len(z) == 0:
        return np.zeros(6)
    P = p66(rot_cov, pos_cov)
    S = h @ P @ h.T + np.diag(r)
    if len(z) == 1:
        S = S + 1e-4
    return P @ h.T @ np.linalg.solve(S, z)


def boxplus(R, p, delta):
    return np.asarray(R) @ synth.exp_so3(delta[:3]), np.asarray(p) + delta[3:]


def load_fixture():
    return dict(np.load(GOLD))
