"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson3_scan_match_ref.so: the UNMODIFIED lesson3 scan-to-scan
node, reference/lesson3/src/scan_match_plicp.cc, compiled where it lies against the ROS and CSM stand-ins under
oracle/shim/ by oracle/ref_lesson3_scan_match.cpp, with sm_icp answered by oracle/plicp_oracle.c.  Its class has the
odometry node's name (oracle/ref_lesson3.py), so it is a library of its own.  `build(ref)` makes the library from a
checkout of the original project; where it is absent the tests replay its recorded answers (tests/reference_record.py).
Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_PATH = os.path.join(_HERE, "_ref", "liblesson3_scan_match_ref.so")
# the flags of oracle/Makefile's builds: x86-64 baseline, no -march, no FMA contraction
CXXFLAGS = ["-std=c++17", "-O2", "-fPIC", "-w", "-ffp-contract=off"]
CFLAGS = ["-std=c11", "-O2", "-fPIC", "-w", "-ffp-contract=off"]
_SHIM = ["ros/ros.h", "sensor_msgs/LaserScan.h", "geometry_msgs/messages.h", "geometry_msgs/TwistStamped.h",
         "tf2/LinearMath/Transform.h", "tf2/utils.h", "tf2_ros/transform_listener.h", "tf2_ros/transform_broadcaster.h",
         "csm/csm_all.h"]
_lib = None


def build(ref: str) -> str:
    srcs = [os.path.join(ref, "lesson3", "src", "scan_match_plicp.cc"),
            os.path.join(ref, "lesson3", "include", "lesson3", "scan_match_plicp.h")]
    drv, orc = os.path.join(_HERE, "ref_lesson3_scan_match.cpp"), os.path.join(_HERE, "plicp_oracle.c")
    deps = srcs + [drv, orc, os.path.join(_ROOT, "include", "b200slam.h")] + [os.path.join(_HERE, "shim", h) for h in _SHIM]
    if not os.path.exists(_PATH) or any(os.path.getmtime(d) > os.path.getmtime(_PATH) for d in deps):
        os.makedirs(os.path.dirname(_PATH), exist_ok=True)
        tmp = _PATH + f".{os.getpid()}.tmp"
        obj = tmp + ".o"
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-c", orc, "-o", obj])
        subprocess.check_call([os.environ.get("CXX", "g++")] + CXXFLAGS +
                              ["-shared", "-I" + os.path.join(_HERE, "shim"),
                               "-I" + os.path.abspath(ref),
                               "-I" + os.path.join(os.path.abspath(ref), "lesson3", "include"), drv, obj, "-o", tmp,
                               "-lm"])
        os.remove(obj)
        os.replace(tmp, _PATH)
    return _PATH


def available() -> bool:
    return os.path.exists(_PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_PATH)
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
