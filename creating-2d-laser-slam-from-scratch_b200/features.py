"""ctypes harness over the C ABI — lesson1: corner-feature extraction (LaserScan::ScanCallback, feature_detection.cc:77-179)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .matcher import check, lib

MAX_BEAMS = 1500  # B2S_FEATURE_MAX_BEAMS
_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        fp = C.POINTER(C.c_float)
        L.b2s_feature_detect.argtypes = [C.c_int, C.c_int, fp, C.c_float, fp, C.POINTER(C.c_int32), fp, C.c_int,
                                         C.c_void_p]
        _bound = True
    return L


def detect(ranges, edge_threshold=1.0, want_curvature=True, device=0, stream=None):
    """ranges [batch][n] (or one scan [n]) -> (out_ranges [batch][n], count [batch], curvature [batch][n] or None).
    count is -1 for a scan with a NaN curvature."""
    L = _bind()
    r = np.ascontiguousarray(np.atleast_2d(ranges), np.float32)
    if r.ndim != 2:
        raise ValueError("ranges must be [batch][n]")
    batch, n = r.shape
    out = np.zeros((batch, n), np.float32)
    cnt = np.zeros(batch, np.int32)
    curv = np.zeros((batch, n), np.float32) if want_curvature else None
    fp = C.POINTER(C.c_float)
    check(L.b2s_feature_detect(batch, n, r.ctypes.data_as(fp), edge_threshold, out.ctypes.data_as(fp),
                               cnt.ctypes.data_as(C.POINTER(C.c_int32)), None if curv is None else curv.ctypes.data_as(fp),
                               device, C.c_void_p(stream) if stream else None))
    return out, cnt, curv
