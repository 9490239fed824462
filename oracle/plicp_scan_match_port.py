"""TEST INFRASTRUCTURE — ctypes binding of oracle/libplicp_scan_match_oracle.so: the plain-C CPU restatement of lesson3's
scan-to-scan node (plicp_scan_match_oracle.c) together with the PL-ICP restatement it calls (plicp_oracle.c), a library
of its own built by oracle/recipes.py.  Only tests/, __graft_entry__ and tools/ may import this module; the product
never does.
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
        L = C.CDLL(recipes.build("libplicp_scan_match_oracle.so"))
        L.orc_plicp_scan_match.restype = None
        L.orc_plicp_scan_match.argtypes = [C.POINTER(abi.IcpParams), C.c_int, C.c_float, C.c_float, C.c_int,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def scan_match(params: abi.IcpParams, angle_min, angle_increment, ranges, limits) -> np.ndarray:
    """orc_plicp_scan_match over one recording from a fresh node.  angle_min, angle_increment float32, ranges [S][n]
    float32, limits [S][2] float32 (range_min, range_max of each scan) -> structured array [S] of
    plicp.SCAN_MATCH_STEP_DTYPE, as b2s_plicp_scan_match_process fills it."""
    r = np.ascontiguousarray(ranges, np.float32)
    lm = np.ascontiguousarray(limits, np.float32)
    assert r.ndim == 2 and lm.shape == (len(r), 2)
    out = np.zeros(len(r), plicp.SCAN_MATCH_STEP_DTYPE)
    lib().orc_plicp_scan_match(C.byref(params), r.shape[1], float(angle_min), float(angle_increment), len(r),
                               r.ctypes.data, lm.ctypes.data, out.ctypes.data)
    return out
