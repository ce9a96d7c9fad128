"""Candidate poses and their records for lk_score_poses: the record (include/legkilo_b200.h: LK_SCORE_*) restated in
float64 from per-point rows (lk_debug_residuals, or the CPU oracle's debug rows), the filter a pose stands for, and the
fixture of tests/golden/ref_score_poses.npz (tests/golden/make_ref_score_golden.py).

Shared by tests/golden/make_ref_score_golden.py, tests/test_score_poses_golden.py (CPU) and tests/test_gpu_score_poses.py."""
import os

import numpy as np

from legkilo_b200 import abi, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_score_poses.npz")
IU = np.triu_indices(6)

# the theta / position blocks of P every scored pose shares: non-isotropic, so their symmetric parts matter
ROT_COV = synth.exp_so3((0.3, 0.2, -0.4)) @ np.diag([2e-6, 5e-6, 8e-6]) @ synth.exp_so3((0.3, 0.2, -0.4)).T
POS_COV = synth.exp_so3((-0.5, 0.1, 0.7)) @ np.diag([4e-6, 1e-6, 9e-6]) @ synth.exp_so3((-0.5, 0.1, 0.7)).T


def pose_state(R, p):
    """The filter state a pose stands for: State::State() (eskf.cc:5-16) at attitude R and position p."""
    x = abi.default_states(1)
    x["rot"][0] = np.asarray(R, np.float64).ravel()
    x["pos"][0] = p
    return x


def pose_cov(rot_cov=ROT_COV, pos_cov=POS_COV):
    """P0 whose theta / position blocks are rot_cov / pos_cov (the only blocks the rows read)."""
    P = 1e-6 * np.eye(30)
    P[:3, :3] = rot_cov
    P[3:6, 3:6] = pos_cov
    return P.ravel().copy()


def row_record(ok, h, z, R):
    """float64 record of per-point rows, and per entry the sum of the absolute values of its terms (its scale)."""
    m = np.asarray(ok).astype(bool)
    h, z, R = np.asarray(h)[m], np.asarray(z)[m], np.asarray(R)[m]
    hh = (h[:, :, None] * h[:, None, :])[:, IU[0], IU[1]] / R[:, None]
    terms = np.concatenate([hh, h * (z / R)[:, None], R[:, None], np.ones((len(z), 1)), (z * z / R)[:, None]], 1)
    rec = np.zeros(abi.SCORE_STRIDE)
    scale = np.zeros(abi.SCORE_STRIDE)
    rec[:30] = terms.sum(0)
    scale[:30] = np.abs(terms).sum(0)
    return rec, scale


def record_err(rec, ref, scale):
    """Largest difference of two records, each entry in units of its scale (the size of its terms)."""
    rec, ref, scale = np.asarray(rec), np.asarray(ref), np.asarray(scale)
    return float(np.max(np.abs(rec - ref) / np.maximum(scale, 1e-300)))


def grid_poses(R0, p0, yaws, offsets):
    """Candidate poses around (R0, p0): yaw about the world z axis times the guess, position guess + offset."""
    rots, poss = [], []
    for yw in yaws:
        Rz = synth.exp_so3((0.0, 0.0, yw))
        for d in offsets:
            rots.append(Rz @ R0)
            poss.append(np.asarray(p0, np.float64) + d)
    return np.array(rots), np.array(poss)


def load_fixture():
    d = dict(np.load(GOLD))
    return d
