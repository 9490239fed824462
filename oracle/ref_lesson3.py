"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson3_ref.so: the UNMODIFIED lesson3 odometry node,
reference/lesson3/src/plicp_odometry.cc, compiled where it lies against the ROS, tf2 and CSM stand-ins under oracle/shim/
by oracle/ref_lesson3.cpp, with sm_icp answered by oracle/plicp_oracle.c, built by oracle/recipes.py from a
checkout of the original project; where it is absent the tests replay its recorded answers (tests/reference_record.py).
Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

from oracle import recipes

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_NAME = "_ref/liblesson3_ref.so"
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
        L.ref_plicp_clear_params.argtypes = []
        L.ref_plicp_clear_params.restype = None
        L.ref_plicp_param.argtypes = [C.c_char_p, C.c_double]
        L.ref_plicp_param.restype = None
        L.ref_plicp_new.argtypes = [dp]
        L.ref_plicp_new.restype = None
        L.ref_plicp_scan.argtypes = [C.c_uint32, C.c_uint32, fp, C.c_int, fp, C.c_void_p]
        L.ref_plicp_scan.restype = C.c_int
        _lib = L
    return _lib


def run(params: dict, mount, fields, ranges, stamps):
    """A fresh node with the parameter-server values `params` (name -> number) and the laser mount (translation xyz +
    quaternion xyzw) over one recording.  fields = (angle_min, angle_increment, range_min, range_max) float32,
    ranges [S][n] float32, stamps [S][2].  -> structured array [S] of the package's plicp.STEP_DTYPE (reference_scan is
    the index of the key frame each scan was matched against, tracked from the keyframe flags)."""
    L = lib()
    sys.path.insert(0, _ROOT) if _ROOT not in sys.path else None
    import importlib
    dtype = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp").STEP_DTYPE
    L.ref_plicp_clear_params()
    for k, v in params.items():
        L.ref_plicp_param(k.encode(), float(v))
    m = np.ascontiguousarray(mount, np.float64)
    L.ref_plicp_new(m.ctypes.data_as(C.POINTER(C.c_double)))
    f = np.ascontiguousarray(fields, np.float32)
    r = np.ascontiguousarray(ranges, np.float32)
    out = np.zeros(len(r), dtype)
    kf = -1
    for s in range(len(r)):
        rc = L.ref_plicp_scan(int(stamps[s][0]), int(stamps[s][1]), f.ctypes.data_as(C.POINTER(C.c_float)), r.shape[1],
                              r[s].ctypes.data_as(C.POINTER(C.c_float)), out[s:s + 1].ctypes.data)
        if rc != 0:
            raise RuntimeError("the lesson3 node threw (a CSM switch the stand-in refuses)")
        if out[s]["published"]:
            out[s]["reference_scan"] = kf
        if out[s]["keyframe"]:
            kf = s
    return out
