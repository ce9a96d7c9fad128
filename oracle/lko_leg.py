"""oracle/lko_leg.py — TEST INFRASTRUCTURE ONLY.

ctypes wrapper over oracle/leg/liblko_leg.so, the CPU restatement of the reference's leg-kinematics step
(ContactDetector / Kinematics of legkilo/src/preprocess/kinematics.{h,cc} and the redundancy drop of
RosInterface::kinematicImuCallBack). Same buffers as lk_leg_kinematics; pinned against the reference by lkref_leg.py.
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

_SO = os.path.join(_HERE, "leg", "liblko_leg.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "leg")])
        L = _LIB = C.CDLL(_SO)
        L.lko_leg_kinematics.restype = C.c_uint32
        L.lko_leg_kinematics.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    return _LIB


def leg_kinematics(states, cfg, track=None, redundancy=True):
    """Same contract as legkilo_b200.Engine.leg_kinematics: returns (kin samples, new abi.LkLegTrack)."""
    states = np.ascontiguousarray(states, abi.LEG_STATE_DTYPE)
    lc = cfg if isinstance(cfg, abi.LkLegCfg) else abi.leg_cfg(cfg)
    tr = abi.leg_track_default()
    if track is not None:
        C.memmove(C.byref(tr), C.byref(track), C.sizeof(tr))
    out = np.zeros(len(states), abi.KINIMU_DTYPE)
    m = lib().lko_leg_kinematics(C.byref(lc), states.ctypes.data_as(C.c_void_p), len(states), int(bool(redundancy)),
                                 C.byref(tr), out.ctypes.data_as(C.c_void_p))
    return out[:m].copy(), tr
