"""oracle/lkref_decode.py — TEST INFRASTRUCTURE ONLY.

ctypes wrapper over oracle/_ref/liblkref_decode.so: the reference's OWN legkilo/src/preprocess/lidar_processing.cc,
compiled unmodified from the reference sources over stand-in headers (oracle/ref_decode/Makefile), fed one
sensor_msgs::PointCloud2 per call. It pins lko_decode.decode_pointcloud2 (tests/test_decode_oracle.py), and
tests/golden/make_ref_decode_golden.py freezes its outputs for boxes without the reference sources.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "liblkref_decode.so")
_REF = "/root/reference/legkilo/src"
_LIB = None


def available() -> bool:
    """True when the library is built, or can be built here (needs the reference sources)."""
    return os.path.exists(_SO) or os.path.isdir(_REF)


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-s", "-C", os.path.join(_HERE, "ref_decode")])
        L = _LIB = C.CDLL(_SO)
        L.lkref_decode_pointcloud2.restype = C.c_uint32
        L.lkref_decode_pointcloud2.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_float, C.c_int32, C.c_double,
                                               C.c_double] + [C.c_void_p] * 4
    return _LIB


def decode_pointcloud2(data, layout, blind, filter_num, time_scale, stamp=0.0):
    """One reference LidarProcessing::processing of a message with these point bytes and header stamp; layout =
    abi.LkPc2Layout. Returns (float4 points, intensity, lidar_begin_time_, lidar_end_time_); NaN times for no points."""
    data = np.ascontiguousarray(data, np.uint8).reshape(-1)
    n = data.size // layout.point_step
    pts = np.zeros((n, 4), np.float32); inten = np.zeros(n, np.float32)
    b = C.c_double(); e = C.c_double()
    m = lib().lkref_decode_pointcloud2(data.ctypes.data_as(C.c_void_p), n, C.byref(layout), blind, filter_num, time_scale,
                                       stamp, pts.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p), C.byref(b),
                                       C.byref(e))
    return pts[:m].copy(), inten[:m].copy(), b.value, e.value
