"""oracle/lko_insert.py — TEST INFRASTRUCTURE ONLY.

ctypes wrapper over oracle/insert/liblko_insert.so: the CPU restatement of oracle/liblko.so (same sources) plus
lko_map_insert, the restatement of lk_map_insert (calcBodyCov and the placement of KILO.cc:216-228 at explicit poses,
then UpdateVoxelMap, set by set). Pinned against the reference by lkref_insert.py.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(_HERE, "..", "leg-kilo_b200", "python"))
from legkilo_b200 import abi  # noqa: E402  (POD struct mirrors only)

_SO = os.path.join(_HERE, "insert", "liblko_insert.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "insert")])
        L = _LIB = C.CDLL(_SO)
        vp = C.c_void_p
        L.lko_create.restype = vp
        L.lko_create.argtypes = [vp] * 4
        L.lko_destroy.argtypes = [vp]
        L.lko_build_voxel_map.argtypes = [vp, vp, vp, C.c_size_t, vp, vp, vp]
        L.lko_map_export.restype = C.c_int
        L.lko_map_export.argtypes = [vp, vp, C.c_size_t, vp]
        L.lko_map_import.restype = C.c_int
        L.lko_map_import.argtypes = [vp, vp, C.c_size_t]
        L.lko_map_insert.argtypes = [vp, C.c_uint32] + [vp] * 6
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def map_insert_args(pts, set_offsets, rot, pos, rot_cov, pos_cov):
    """The contiguous buffers of a map_insert call: float32 [n, 4], uint32 [n_sets + 1], float64 rows per set."""
    so = np.ascontiguousarray(set_offsets, np.uint32)
    n = len(so) - 1
    return (np.ascontiguousarray(pts, np.float32).reshape(-1, 4), so,
            *(np.ascontiguousarray(a, np.float64).reshape(n, k) for a, k in ((rot, 9), (pos, 3), (rot_cov, 9), (pos_cov, 9))))


class Oracle:
    """The oracle's VoxelMapManager with the extrinsics of `cfg`: what lk_map_insert needs of lko.Oracle."""

    def __init__(self, cfg: dict):
        self.cfg = cfg
        self._ec, self._mc = abi.eskf_cfg(cfg), abi.map_cfg(cfg)
        self._R, self._t = abi.extrinsics(cfg)
        self.h = lib().lko_create(C.byref(self._ec), C.byref(self._mc), _p(self._R), _p(self._t))

    def __del__(self):
        if getattr(self, "h", None):
            lib().lko_destroy(self.h)
            self.h = None

    def build_voxel_map(self, xyz_world, xyz_body, R, rot_cov, pos_cov):
        xyz_world = np.ascontiguousarray(xyz_world, np.float32)
        xyz_body = np.ascontiguousarray(xyz_body, np.float32)
        R, rot_cov, pos_cov = (np.ascontiguousarray(a, np.float64) for a in (R, rot_cov, pos_cov))
        lib().lko_build_voxel_map(self.h, _p(xyz_world), _p(xyz_body), len(xyz_world), _p(R), _p(rot_cov), _p(pos_cov))

    def map_insert(self, pts, set_offsets, rot, pos, rot_cov, pos_cov):
        pts, so, rot, pos, rot_cov, pos_cov = map_insert_args(pts, set_offsets, rot, pos, rot_cov, pos_cov)
        lib().lko_map_insert(self.h, len(so) - 1, _p(pts), _p(so), _p(rot), _p(pos), _p(rot_cov), _p(pos_cov))

    def map_export(self) -> np.ndarray:
        sz = C.c_size_t(0)
        lib().lko_map_export(self.h, None, 0, C.byref(sz))
        buf = np.zeros(sz.value, np.uint8)
        assert lib().lko_map_export(self.h, _p(buf), buf.size, C.byref(sz)) == 0
        return buf

    def map_import(self, blob: np.ndarray):
        blob = np.ascontiguousarray(blob, np.uint8)
        assert lib().lko_map_import(self.h, _p(blob), blob.size) == 0
