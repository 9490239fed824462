"""TEST INFRASTRUCTURE — ctypes binding of oracle/libfeature_oracle.so, the C++ CPU restatement of lesson1's corner picker
(feature_oracle.cpp, LaserScan::ScanCallback, feature_detection.cc:77-179).  It is a library of its own, built from one
C++ file by oracle/recipes.py.  Only tests/, __graft_entry__ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

MAX_BEAMS = 1500
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.build("libfeature_oracle.so"))
        fp = C.POINTER(C.c_float)
        L.orc_feature_detect.argtypes = [C.c_int, fp, C.c_float, fp, fp, C.POINTER(C.c_int32)]
        L.orc_feature_detect.restype = C.c_int
        L.orc_feature_killer_order.argtypes = [C.c_int, C.POINTER(C.c_uint8), fp]
        L.orc_feature_killer_order.restype = None
        _lib = L
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class Result:
    """ranges [batch][n], count [batch] (-1 = NaN curvature), curvature [batch][n], tied [batch] (bit j: sector j's
    cut is tied), heap [batch] (sector sorts that fell back to heap sort)."""

    def __init__(self, batch, n):
        self.ranges = np.zeros((batch, n), np.float32)
        self.curvature = np.zeros((batch, n), np.float32)
        self.count = np.zeros(batch, np.int32)
        self.tied = np.zeros(batch, np.int32)
        self.heap = np.zeros(batch, np.int32)


def detect(ranges, edge_threshold=1.0) -> Result:
    """ScanCallback on every row of ranges [batch][n] (or one scan [n])."""
    r = np.ascontiguousarray(np.atleast_2d(ranges), np.float32)
    batch, n = r.shape
    if n > MAX_BEAMS:
        raise ValueError(f"the node takes at most {MAX_BEAMS} beams")
    L, out = lib(), Result(batch, n)
    info = np.zeros(4, np.int32)
    for b in range(batch):
        rc = L.orc_feature_detect(n, _fp(r[b]), edge_threshold, _fp(out.ranges[b]), _fp(out.curvature[b]),
                                  info.ctypes.data_as(C.POINTER(C.c_int32)))
        assert rc == 0
        assert info[3] == 0, "csrc/introsort.cuh disagrees with std::sort"
        out.count[b], out.tied[b], out.heap[b] = info[0], info[1], info[2]
    return out


def detect_timed(ranges, edge_threshold=1.0) -> float:
    """seconds the restatement takes on every row of ranges [batch][n], without the diagnostics of detect()"""
    import time
    r = np.ascontiguousarray(np.atleast_2d(ranges), np.float32)
    out, curv = np.zeros(r.shape[1], np.float32), np.zeros(r.shape[1], np.float32)
    L = lib()
    t0 = time.perf_counter()
    for b in range(len(r)):
        L.orc_feature_detect(r.shape[1], _fp(r[b]), edge_threshold, _fp(out), _fp(curv), None)
    return time.perf_counter() - t0


def killer_order(n, top=None) -> np.ndarray:
    """values whose order drives this host's std::sort into its heap-sort fallback (McIlroy's adversary); elements
    where `top` is true are fixed as equal maxima (n + 1) before the adversary orders the rest"""
    out = np.zeros(n, np.float32)
    t = None if top is None else np.ascontiguousarray(top, np.uint8)
    lib().orc_feature_killer_order(n, None if t is None else t.ctypes.data_as(C.POINTER(C.c_uint8)), _fp(out))
    return out
