"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson1_ref.so: the UNMODIFIED lesson1 node,
reference/lesson1/src/feature_detection.cc, compiled where it lies against the ROS stand-in under oracle/shim/ by
oracle/ref_lesson1.cpp, built by oracle/recipes.py from a checkout of the original project; where it is absent the
tests replay its recorded answers (tests/reference_record.py).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/liblesson1_ref.so"
MAX_BEAMS = 1500
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        L.ref_feature_detect.argtypes = [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        L.ref_feature_detect.restype = C.c_int
        _lib = L
    return _lib


def detect(ranges) -> np.ndarray:
    """The node's published corner_scan.ranges [batch][1500] for every row of ranges [batch][n] (edge_threshold 1.0)."""
    r = np.ascontiguousarray(np.atleast_2d(ranges), np.float32)
    out = np.zeros((len(r), MAX_BEAMS), np.float32)
    fp = C.POINTER(C.c_float)
    for b in range(len(r)):
        rc = lib().ref_feature_detect(r.shape[1], r[b].ctypes.data_as(fp), out[b].ctypes.data_as(fp))
        if rc != 0:
            raise ValueError(f"the node refuses a scan of {r.shape[1]} beams")
    return out
