"""TEST INFRASTRUCTURE — ctypes binding of oracle/libplicp_odometry_oracle.so: the plain-C CPU restatement of lesson3's
odometry node (plicp_odometry_oracle.c) together with the PL-ICP restatement it calls (plicp_oracle.c), a library of its
own built by oracle/recipes.py.  Only tests/, __graft_entry__ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib

import numpy as np

from oracle import recipes

abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")
plicp = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp")

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.build("libplicp_odometry_oracle.so"))
        L.orc_plicp_odometry.restype = None
        L.orc_plicp_odometry.argtypes = [C.POINTER(abi.PlicpOdomParams), C.c_int, C.c_float, C.c_float, C.c_float,
                                         C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def odometry(params: abi.PlicpOdomParams, fields, ranges, stamps) -> np.ndarray:
    """orc_plicp_odometry over one recording from a fresh node.  fields = (angle_min, angle_increment, range_min,
    range_max) as float32, ranges [S][n] float32, stamps [S][2] (sec, nsec) -> structured array [S] of
    plicp.STEP_DTYPE, as b2s_plicp_odom_process fills it."""
    r = np.ascontiguousarray(ranges, np.float32)
    s = np.ascontiguousarray(stamps, np.uint32)
    assert r.ndim == 2 and s.shape == (len(r), 2)
    out = np.zeros(len(r), plicp.STEP_DTYPE)
    lib().orc_plicp_odometry(C.byref(params), r.shape[1], *map(float, fields), len(r), r.ctypes.data, s.ctypes.data,
                             out.ctypes.data)
    return out
