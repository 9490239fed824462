"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson3_scan_match_ref.so: the UNMODIFIED lesson3 scan-to-scan
node, reference/lesson3/src/scan_match_plicp.cc, compiled where it lies against the ROS and CSM stand-ins under
oracle/shim/ by oracle/ref_lesson3_scan_match.cpp, with sm_icp answered by oracle/plicp_oracle.c.  Its class has the
odometry node's name (oracle/ref_lesson3.py), so it is a library of its own, built by oracle/recipes.py from a
checkout of the original project; where it is absent the tests replay its recorded answers (tests/reference_record.py).
Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C
import importlib
import os
import sys

import numpy as np

from oracle import recipes

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_NAME = "_ref/liblesson3_scan_match_ref.so"
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        fp = C.POINTER(C.c_float)
        L.ref_sm_clear_params.argtypes = []
        L.ref_sm_clear_params.restype = None
        L.ref_sm_param.argtypes = [C.c_char_p, C.c_double]
        L.ref_sm_param.restype = None
        L.ref_sm_new.argtypes = []
        L.ref_sm_new.restype = None
        L.ref_sm_scan.argtypes = [C.c_uint32, C.c_uint32, fp, C.c_int, fp, C.c_void_p]
        L.ref_sm_scan.restype = C.c_int
        _lib = L
    return _lib


def run(params: dict, angle_min, angle_increment, ranges, limits):
    """A fresh node with the parameter-server values `params` (name -> number) over one recording: ranges [S][n]
    float32, limits [S][2] float32 (range_min, range_max of each scan).  -> structured array [S] of the package's
    plicp.SCAN_MATCH_STEP_DTYPE.  Raises RuntimeError when the node throws (a CSM switch the stand-in refuses)."""
    L = lib()
    sys.path.insert(0, _ROOT) if _ROOT not in sys.path else None
    dtype = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp").SCAN_MATCH_STEP_DTYPE
    L.ref_sm_clear_params()
    for k, v in params.items():
        L.ref_sm_param(k.encode(), float(v))
    L.ref_sm_new()
    r = np.ascontiguousarray(ranges, np.float32)
    lm = np.ascontiguousarray(limits, np.float32)
    out = np.zeros(len(r), dtype)
    for s in range(len(r)):
        f = np.array([angle_min, angle_increment, lm[s][0], lm[s][1]], np.float32)
        rc = L.ref_sm_scan(0, s, f.ctypes.data_as(C.POINTER(C.c_float)), r.shape[1],
                           r[s].ctypes.data_as(C.POINTER(C.c_float)), out[s:s + 1].ctypes.data)
        if rc != 0:
            raise RuntimeError("the lesson3 scan-match node threw (a CSM switch the stand-in refuses)")
    return out
