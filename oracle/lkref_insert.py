"""oracle/lkref_insert.py — TEST INFRASTRUCTURE ONLY.

ctypes wrapper over oracle/_ref/liblkref_insert.so: the reference's own eskf.cc / voxel_map.cc / KILO.cc with the harness
of oracle/ref plus lkref_map_insert (oracle/ref_insert/), which places point sets at explicit poses with the reference's
calcBodyCov and SKEW_SYM_MATRIX and hands them to its UpdateVoxelMap. Pins oracle/lko_insert.py (lk_map_insert's oracle).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(_HERE, "..", "leg-kilo_b200", "python"))
sys.path.insert(0, _HERE)
import lko_insert  # noqa: E402
from legkilo_b200 import abi  # noqa: E402  (POD struct mirrors only)

_SO = os.path.join(_HERE, "_ref", "liblkref_insert.so")
_LIB = None


def available() -> bool:
    """True when the library is built, or can be built here (needs /root/reference)."""
    return os.path.exists(_SO) or os.path.isdir("/root/reference/legkilo/src")


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "ref_insert")])
        L = _LIB = C.CDLL(_SO)
        vp = C.c_void_p
        L.lkref_create.restype = vp
        L.lkref_create.argtypes = [vp, vp, vp, vp, C.c_int, C.c_double]
        L.lkref_destroy.argtypes = [vp]
        L.lkref_set_runtime.argtypes = [vp, C.c_double, C.c_int]
        L.lkref_build_voxel_map.argtypes = [vp, vp, vp, C.c_size_t, vp, vp, vp]
        L.lkref_map_export.restype = C.c_int
        L.lkref_map_export.argtypes = [vp, vp, C.c_size_t, vp]
        L.lkref_map_insert.argtypes = [vp, C.c_uint32] + [vp] * 6
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Reference:
    """One legkilo::KILO built from the same config dict as lko_insert.Oracle: its map, built and updated."""

    def __init__(self, cfg: dict):
        ec, mc = abi.eskf_cfg(cfg), abi.map_cfg(cfg)
        R, t = abi.extrinsics(cfg)
        self.h = lib().lkref_create(C.byref(ec), C.byref(mc), _p(R), _p(t), 1, 9.81)
        lib().lkref_set_runtime(self.h, 1.0, 1)

    def __del__(self):
        if getattr(self, "h", None):
            lib().lkref_destroy(self.h)
            self.h = None

    def build_voxel_map(self, xyz_world, xyz_body, R, rot_cov, pos_cov):
        xyz_world = np.ascontiguousarray(xyz_world, np.float32)
        xyz_body = np.ascontiguousarray(xyz_body, np.float32)
        R, rot_cov, pos_cov = (np.ascontiguousarray(a, np.float64) for a in (R, rot_cov, pos_cov))
        lib().lkref_build_voxel_map(self.h, _p(xyz_world), _p(xyz_body), len(xyz_world), _p(R), _p(rot_cov), _p(pos_cov))

    def map_insert(self, pts, set_offsets, rot, pos, rot_cov, pos_cov):
        pts, so, rot, pos, rot_cov, pos_cov = lko_insert.map_insert_args(pts, set_offsets, rot, pos, rot_cov, pos_cov)
        lib().lkref_map_insert(self.h, len(so) - 1, _p(pts), _p(so), _p(rot), _p(pos), _p(rot_cov), _p(pos_cov))

    def map_export(self) -> np.ndarray:
        sz = C.c_size_t(0)
        lib().lkref_map_export(self.h, None, 0, C.byref(sz))
        buf = np.zeros(sz.value, np.uint8)
        assert lib().lkref_map_export(self.h, _p(buf), buf.size, C.byref(sz)) == 0
        return buf
