"""TEST INFRASTRUCTURE — ctypes binding of oracle/libdeskew_node_oracle.so: the plain-C CPU restatement of lesson5's
whole de-skew node over a recording (deskew_node_oracle.c) together with the per-scan restatement it calls
(deskew_oracle.c), a library of its own built with the flags of oracle/Makefile.  Only tests/, __graft_entry__ and
tools/ may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib
import os
import subprocess

import numpy as np

deskew = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = [os.path.join(_HERE, f) for f in ("deskew_node_oracle.c", "deskew_oracle.c")]
_HDR = os.path.join(_HERE, "linear_math.h")
_LIB = os.path.join(_HERE, "libdeskew_node_oracle.so")
# the flags of oracle/Makefile: x86-64 baseline, no FMA contraction
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wextra", "-D_DEFAULT_SOURCE"]
QUEUE_LENGTH = 2000
_lib = None


def build(force: bool = False) -> str:
    deps = _SRC + [_HDR, os.path.abspath(__file__)]
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
        tmp = _LIB + f".{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-shared"] + _SRC + ["-o", tmp, "-lm"])
        os.replace(tmp, _LIB)  # atomic: a concurrent reader sees the old library or the new one
    return _LIB


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp = C.c_void_p
        L.orc_deskew_node.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, vp, vp, C.c_int, vp,
                                      C.c_int, vp, vp, vp, vp, vp, vp]
        L.orc_deskew_node.restype = C.c_int
        _lib = L
    return _lib


def node(use_imu, use_odom, angle_min, angle_increment, scans, ranges, imu, odom, tables=False):
    """One recording through the restated node.  scans / imu / odom: the numpy record arrays of
    deskew.recording_arrays; ranges [S][n] float32.  -> dict of status [S], state [S] (deskew.STATE_DTYPE), xyz
    [S, n, 3], poses [S, 2, 6] and, with tables, imu [S, 4, 2000]."""
    r = np.ascontiguousarray(ranges, np.float32)
    S, n = r.shape
    status = np.zeros(S, np.int32)
    state = np.zeros(S, deskew.STATE_DTYPE)
    xyz = np.zeros((S, n, 3), np.float32)
    poses = np.zeros((S, 2, 6))
    tab = np.zeros((S, 4, QUEUE_LENGTH)) if tables else None
    assert lib().orc_deskew_node(int(use_imu), int(use_odom), float(angle_min), float(angle_increment), n, S,
                                 scans.ctypes.data, r.ctypes.data, len(imu), imu.ctypes.data if len(imu) else None,
                                 len(odom), odom.ctypes.data if len(odom) else None, status.ctypes.data,
                                 state.ctypes.data, xyz.ctypes.data, poses.ctypes.data,
                                 tab.ctypes.data if tables else None) == 0
    out = dict(status=status, state=state, xyz=xyz, poses=poses)
    if tables:
        out["imu"] = tab
    return out
