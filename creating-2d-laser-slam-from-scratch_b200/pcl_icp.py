"""ctypes harness over the C ABI — lesson2: batched PCL point-to-point ICP (ScanMatchWithICP, scan_match_icp.cc:135-164)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .matcher import check, lib

_bound = False

RESULT_DTYPE = np.dtype([("x", "<f4", 3), ("converged", "<i4"), ("iterations", "<i4"), ("n_correspondences", "<i4"),
                         ("fitness_score", "<f8")])


def _bind():
    global _bound
    L = lib()
    if not _bound:
        fp = C.POINTER(C.c_float)
        L.b2s_pcl_icp_align.argtypes = [C.POINTER(abi.PclIcpParams), C.c_int, C.c_int, fp, C.c_float, C.c_float,
                                        C.c_float, C.c_float, C.c_int, C.POINTER(C.c_int32), fp, C.c_int, C.c_void_p,
                                        C.POINTER(abi.PclIcpResult)]
        _bound = True
    return L


def align(params: abi.PclIcpParams, ranges, angle_min, angle_increment, range_min, range_max, pairs=None,
          guesses=None, device=0, stream=None):
    """ranges [n_scans][n]; pairs [n_pairs][2] (source, target) or None for the consecutive pairs (i - 1, i);
    guesses [n_pairs][3] or None.  -> structured array [n_pairs] (x, converged, iterations, n_correspondences,
    fitness_score)."""
    L = _bind()
    r = np.ascontiguousarray(ranges, np.float32)
    if r.ndim != 2:
        raise ValueError("ranges must be [n_scans][n]")
    n_scans, n = r.shape
    p = None if pairs is None else np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    n_pairs = n_scans - 1 if p is None else len(p)
    g = None if guesses is None else np.ascontiguousarray(guesses, np.float32).reshape(-1, 3)
    if g is not None and len(g) != n_pairs:
        raise ValueError("one guess per pair")
    res = (abi.PclIcpResult * max(n_pairs, 1))()
    fp = C.POINTER(C.c_float)
    check(L.b2s_pcl_icp_align(C.byref(params), n_scans, n, r.ctypes.data_as(fp), angle_min, angle_increment,
                              range_min, range_max, n_pairs, None if p is None else p.ctypes.data_as(C.POINTER(C.c_int32)),
                              None if g is None else g.ctypes.data_as(fp), device,
                              C.c_void_p(stream) if stream else None, res))
    return np.frombuffer(res, dtype=RESULT_DTYPE, count=n_pairs).copy()
