"""Shared fixtures-as-functions for the parity tests: scenes from legkilo_b200.synth fed, unchanged,
to the CPU oracle and to the CUDA library."""
import os

import numpy as np

import lko
from legkilo_b200 import abi, synth


def planar_scene(cfg_name="leg_fusion", n=2048, half_extent=20.0, seed_stream=2, rotvec=(2e-3, -1e-3, 3e-3),
                 trans=(0.02, -0.01, 0.03)):
    cfg = abi.CONFIGS[cfg_name]
    R, t = abi.extrinsics(cfg)
    pw, pb = synth.planar_map_points(half_extent=half_extent, ext_R=R, ext_t=t)
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw, pb)
    blob = o.map_export()
    pts = synth.planar_scan(n=n, ext_R=R, ext_t=t, stream=seed_stream, rotvec=rotvec, trans=trans)
    return cfg, blob, pts


def box_scene(cfg_name="leg_fusion", lidar=None, ground_half_extent=20.0, batch=1, rot_sigma=2e-3, trans_sigma=0.02,
              streaming=False, stream0=100):
    """Box room, map built by the ORACLE's BuildVoxelMap over a small ground patch."""
    cfg = abi.CONFIGS[cfg_name]
    R, t = abi.extrinsics(cfg)
    sc = synth.BoxScene(ground_half_extent=ground_half_extent)
    pw, pb = sc.map_points(ext_R=R, ext_t=t)
    o = lko.Oracle(cfg)
    o.build_voxel_map(pw, pb)
    blob = o.map_export()
    lidar = lidar or synth.VLP16
    rv, tv = synth.random_poses(batch, rot_sigma, trans_sigma, stream=stream0)
    scans = [sc.scan(rotvec=rv[i], trans=tv[i], ext_R=R, ext_t=t, blind=cfg["blind"], stream=stream0 + 1 + i,
                     streaming=streaming, **lidar) for i in range(batch)]
    return cfg, blob, scans


# ---- comparing filters -------------------------------------------------------------------------------------------------
# The blocks of P differ in scale by orders of magnitude (after a few dozen predicts the imu_w / imu_a variances are ~1e4
# times the pose variances), so an error measured against P's largest entry hides the pose block. Both comparisons below
# measure each entry in the filter's own units instead: covariances in correlation units, states in standard deviations.

BLOCKS = ("theta", "pos", "vel", "ba", "bw", "grav", "imu_a", "imu_w", "bv", "contact")  # the 30-vector's order


def state_name(k):
    return f"{BLOCKS[k // 3]}.{'xyz'[k % 3]}"


class Err(float):
    """A comparison's worst value, with the entry where it was reached: `assert e < tol, e` names it."""

    def __new__(cls, value, where):
        e = super().__new__(cls, value)
        e.where = where
        return e

    def __repr__(self):
        return f"{float(self):.3e} at {self.where}"

    __str__ = __repr__


def _sd(P_ref):
    d = np.diag(np.asarray(P_ref, np.float64).reshape(30, 30))
    bad = np.flatnonzero(~(d > 0))
    assert len(bad) == 0, f"reference covariance has a non-positive variance at {state_name(int(bad[0]))}: {d[bad[0]]}"
    return np.sqrt(d)


def cov_err(P, P_ref):
    """max_ij |P_ij - Pref_ij| / sqrt(Pref_ii Pref_jj): the error in correlation units. Reads only the diagonal of P_ref,
    so it holds for asymmetric (skewed) covariances too."""
    sd = _sd(P_ref)
    e = np.abs(np.asarray(P, np.float64).reshape(30, 30) - np.asarray(P_ref, np.float64).reshape(30, 30)) / np.outer(sd, sd)
    i, j = np.unravel_index(int(np.argmax(e)), e.shape)
    return Err(e[i, j], f"P[{state_name(i)}, {state_name(j)}]")


def state_err(x, x_ref, P_ref):
    """max_k |(x [-] x_ref)_k| / sqrt(Pref_kk): the error in posterior standard deviations."""
    e = np.abs(lko.boxminus(x, x_ref)) / _sd(P_ref)
    k = int(np.argmax(e))
    return Err(e[k], f"x[{state_name(k)}]")


def check_filter(x, P, x_ref, P_ref, state_tol, cov_tol, what=""):
    """Asserts state_err < state_tol and cov_err < cov_tol, and prints both (pytest -s shows them with the test id) so that
    the tolerances can be restated from measurements."""
    ex, eP = state_err(x, x_ref, P_ref), cov_err(P, P_ref)
    test = os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0]
    print(f"filter-err {test} {what}: state_err {ex!r} cov_err {eP!r}")
    assert ex < state_tol and eP < cov_tol, (what, f"state_err {ex!r} (tol {state_tol:g})", f"cov_err {eP!r} (tol {cov_tol:g})")
    return ex, eP
