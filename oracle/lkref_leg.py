"""oracle/lkref_leg.py — TEST INFRASTRUCTURE ONLY.

ctypes wrapper over oracle/_ref/liblkref_leg.so: the reference's OWN legkilo/src/preprocess/kinematics.cc, compiled
unmodified from the reference sources over stand-in headers (oracle/ref_leg/Makefile), driven from its initial state
with the redundancy rule of RosInterface::kinematicImuCallBack restated. It pins oracle/lko_leg.py
(tests/test_leg_kinematics.py), and tests/golden/make_ref_leg_golden.py freezes its outputs for boxes without the
reference sources.
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

_SO = os.path.join(_HERE, "_ref", "liblkref_leg.so")
_REF = "/root/reference/legkilo/src"
_LIB = None


def available() -> bool:
    """True when the library is built, or can be built here (needs the reference sources)."""
    return os.path.exists(_SO) or os.path.isdir(_REF)


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "ref_leg")])
        L = _LIB = C.CDLL(_SO)
        L.lkref_leg_kinematics.restype = C.c_uint32
        L.lkref_leg_kinematics.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    return _LIB


def leg_kinematics(states, cfg, redundancy=True):
    """One reference Kinematics over `states` from its initial state. Returns (kin samples, abi.LkLegTrack after)."""
    states = np.ascontiguousarray(states, abi.LEG_STATE_DTYPE)
    lc = cfg if isinstance(cfg, abi.LkLegCfg) else abi.leg_cfg(cfg)
    out = np.zeros(len(states), abi.KINIMU_DTYPE)
    tr = abi.LkLegTrack()
    m = lib().lkref_leg_kinematics(C.byref(lc), states.ctypes.data_as(C.c_void_p), len(states), int(bool(redundancy)),
                                   out.ctypes.data_as(C.c_void_p), C.byref(tr))
    return out[:m].copy(), tr
