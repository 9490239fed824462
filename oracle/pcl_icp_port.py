"""TEST INFRASTRUCTURE — ctypes binding of oracle/libpcl_icp_oracle.so, the plain-C CPU restatement of lesson2's ICP
scan matching (pcl_icp_oracle.c, PARITY UNPINNED).  It is a library of its own, built from one C file by
oracle/recipes.py, so that the restatement of lesson2 needs nothing from the other restatements.  Only tests/,
__graft_entry__ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib

import numpy as np

from oracle import recipes

abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.build("libpcl_icp_oracle.so"))
        fp = C.POINTER(C.c_float)
        L.orc_pcl_scan_to_cloud.argtypes = [C.c_int, fp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, fp]
        L.orc_pcl_scan_to_cloud.restype = C.c_int
        L.orc_pcl_icp_align.argtypes = [C.POINTER(abi.PclIcpParams), C.c_int, fp, C.c_int, fp, fp,
                                        C.POINTER(abi.PclIcpResult), C.POINTER(C.c_int)]
        L.orc_pcl_icp_align.restype = None
        _lib = L
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def pcl_scan_to_cloud(ranges, angle_min, angle_increment, range_min, range_max, drop_invalid=False):
    """ConvertScan2PointCloud -> float32 [m, 2] (m = n unless invalid readings are dropped)."""
    r = np.ascontiguousarray(ranges, np.float32)
    xy = np.zeros((len(r), 2), np.float32)
    m = lib().orc_pcl_scan_to_cloud(len(r), _fp(r), angle_min, angle_increment, range_min, range_max,
                                    int(drop_invalid), _fp(xy))
    return xy[:m].copy()


def pcl_icp_align(params, src_ranges, tgt_ranges, angle_min, angle_increment, range_min, range_max, guess=None,
                  corr=False):
    """ScanMatchWithICP for one pair (source = previous scan, target = current scan) -> abi.PclIcpResult, and with
    corr=True also the target index of every source point in the last correspondence search (-1 = rejected)."""
    drop = bool(params.drop_invalid_points)
    s = pcl_scan_to_cloud(src_ranges, angle_min, angle_increment, range_min, range_max, drop)
    t = pcl_scan_to_cloud(tgt_ranges, angle_min, angle_increment, range_min, range_max, drop)
    g = None if guess is None else np.ascontiguousarray(guess, np.float32)
    res = abi.PclIcpResult()
    nn = np.full(max(len(s), 1), -1, np.int32)
    lib().orc_pcl_icp_align(C.byref(params), len(s), _fp(s), len(t), _fp(t), None if g is None else _fp(g),
                            C.byref(res), nn.ctypes.data_as(C.POINTER(C.c_int)))
    return (res, nn[:len(s)]) if corr else res
