"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson1_ref.so: the UNMODIFIED lesson1 node,
reference/lesson1/src/feature_detection.cc, compiled where it lies against the ROS stand-in under oracle/shim/ by
oracle/ref_lesson1.cpp.  `build(ref)` makes the library from a checkout of the original project; where it is absent the
tests replay its recorded answers (tests/reference_record.py).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "_ref", "liblesson1_ref.so")
# the flags of oracle/Makefile's reference builds: x86-64 baseline, no -march, so no FMA contraction
CXXFLAGS = ["-std=c++17", "-O2", "-fPIC", "-w"]
MAX_BEAMS = 1500
_lib = None


def build(ref: str) -> str:
    src = os.path.join(ref, "lesson1", "src", "feature_detection.cc")
    drv = os.path.join(_HERE, "ref_lesson1.cpp")
    shim = [os.path.join(_HERE, "shim", "ros", "ros.h"), os.path.join(_HERE, "shim", "sensor_msgs", "LaserScan.h")]
    if not os.path.exists(_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_PATH) for d in [src, drv] + shim):
        os.makedirs(os.path.dirname(_PATH), exist_ok=True)
        tmp = _PATH + f".{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CXX", "g++")] + CXXFLAGS +
                              ["-shared", "-I" + os.path.join(_HERE, "shim"), "-I" + os.path.abspath(ref), drv, "-o", tmp])
        os.replace(tmp, _PATH)
    return _PATH


def available() -> bool:
    return os.path.exists(_PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_PATH)
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
