"""TEST INFRASTRUCTURE — ctypes binding of oracle/libdeskew_node_oracle.so: the plain-C CPU restatement of lesson5's whole
de-skew node over a recording (deskew_node_oracle.c) together with the per-scan restatement it calls (deskew_oracle.c),
a library of its own built by oracle/recipes.py.  Only tests/, __graft_entry__ and tools/ may import this module; the
product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib

import numpy as np

from oracle import recipes

deskew = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")

QUEUE_LENGTH = 2000
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.build("libdeskew_node_oracle.so"))
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
