"""TEST INFRASTRUCTURE — ctypes binding of oracle/libplicp_scan_match_oracle.so: the plain-C CPU restatement of lesson3's
scan-to-scan node (plicp_scan_match_oracle.c) together with the PL-ICP restatement it calls (plicp_oracle.c), a library
of its own built with the flags of oracle/Makefile.  Only tests/, __graft_entry__ and tools/ may import this module;
the product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib
import os
import subprocess

import numpy as np

abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")
plicp = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp")

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = [os.path.join(_HERE, "plicp_scan_match_oracle.c"), os.path.join(_HERE, "plicp_oracle.c")]
_HDR = os.path.join(os.path.dirname(_HERE), "include", "b200slam.h")
_LIB = os.path.join(_HERE, "libplicp_scan_match_oracle.so")
# the flags of oracle/Makefile: x86-64 baseline, no FMA contraction
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wextra"]
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
