"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson6_ref.so: the UNMODIFIED lesson6 Karto SLAM node,
reference/lesson6/src/karto_slam.cc, compiled where it lies with the unmodified open_karto Karto.cpp / Mapper.cpp against
the ROS, tf and Boost stand-ins under oracle/shim_lesson6/ and oracle/shim/ by oracle/ref_lesson6.cpp, built by
oracle/recipes.py from a checkout of the original project; where it is absent the tests replay its recorded answers
(tests/reference_record.py).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C
import importlib
import os
import sys

import numpy as np

from oracle import recipes

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_NAME = "_ref/liblesson6_ref.so"
MAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_double, C.c_double, C.POINTER(C.c_int8))
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        dp, fp, ip = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32)
        sys.path.insert(0, _ROOT) if _ROOT not in sys.path else None
        ScanSolver = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.mapper").ScanSolver
        L.ref_karto_clear_params.argtypes = []
        L.ref_karto_clear_params.restype = None
        L.ref_karto_param.argtypes = [C.c_char_p, C.c_double]
        L.ref_karto_param.restype = None
        L.ref_karto_param_str.argtypes = [C.c_char_p, C.c_char_p]
        L.ref_karto_param_str.restype = None
        L.ref_karto_set_solver.argtypes = [C.POINTER(ScanSolver)]
        L.ref_karto_set_solver.restype = None
        L.ref_karto_new.argtypes = [dp]
        L.ref_karto_new.restype = C.c_void_p
        L.ref_karto_scan.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, fp, C.c_int, fp, dp, ip, dp, dp, ip, MAP_FN,
                                     C.c_void_p]
        L.ref_karto_scan.restype = C.c_int
        L.ref_karto_scan_count.argtypes = [C.c_void_p]
        L.ref_karto_poses.argtypes = [C.c_void_p, dp]
        L.ref_karto_poses.restype = None
        L.ref_karto_edge_count.argtypes = [C.c_void_p]
        L.ref_karto_edges.argtypes = [C.c_void_p, ip, dp, dp]
        L.ref_karto_edges.restype = None
        _lib = L
    return _lib


def run(params: dict, fields, mount, ranges, stamps, odom, solver=None):
    """A fresh node with the parameter-server values `params` (name -> number or string) over one recording.
    fields = (angle_min, angle_max, angle_increment, range_min, range_max) float32, mount = base_link <- laser
    (translation xyz + quaternion xyzw), ranges [S][n] float32, stamps [S][2], odom [S][7] (NaN = lookup fails),
    solver = a mapper.ScanSolver for use_back_end.  -> dict(state, pose, map_to_odom, map_published, maps, poses, edges):
    maps = [(scan index, dict(width, height, resolution, offset), int8 payload [height][width])], poses / edges = the
    graph at the end."""
    L = lib()
    L.ref_karto_clear_params()
    for k, v in params.items():
        if isinstance(v, str):
            L.ref_karto_param_str(k.encode(), v.encode())
        else:
            L.ref_karto_param(k.encode(), float(v))
    L.ref_karto_set_solver(C.byref(solver) if solver is not None else None)
    m = np.ascontiguousarray(mount, np.float64)
    h = L.ref_karto_new(m.ctypes.data_as(C.POINTER(C.c_double)))
    f = np.ascontiguousarray(fields, np.float32)
    r = np.ascontiguousarray(ranges, np.float32)
    o = np.ascontiguousarray(odom, np.float64)
    S = len(r)
    out = dict(state=np.zeros(S, np.int32), pose=np.zeros((S, 3)), map_to_odom=np.zeros((S, 7)),
               map_published=np.zeros(S, np.int32), maps=[])
    cur = [0]

    def cb(user, w, hgt, res, ox, oy, payload):
        data = np.ctypeslib.as_array(payload, shape=(w * hgt,)).reshape(hgt, w).copy() if w * hgt else \
            np.zeros((hgt, w), np.int8)
        out["maps"].append((cur[0], dict(width=w, height=hgt, resolution=res, offset=np.array([ox, oy])), data))

    fn = MAP_FN(cb)
    st, pub = C.c_int32(), C.c_int32()
    for s in range(S):
        cur[0] = s
        rc = L.ref_karto_scan(h, int(stamps[s][0]), int(stamps[s][1]), f.ctypes.data_as(C.POINTER(C.c_float)), r.shape[1],
                              r[s].ctypes.data_as(C.POINTER(C.c_float)), o[s].ctypes.data_as(C.POINTER(C.c_double)),
                              C.byref(st), out["pose"][s].ctypes.data_as(C.POINTER(C.c_double)),
                              out["map_to_odom"][s].ctypes.data_as(C.POINTER(C.c_double)), C.byref(pub), fn, None)
        if rc != 0:
            raise RuntimeError("the lesson6 node threw")
        out["state"][s], out["map_published"][s] = st.value, pub.value
    n = L.ref_karto_scan_count(h)
    out["poses"] = np.zeros((n, 3))
    if n:
        L.ref_karto_poses(h, out["poses"].ctypes.data_as(C.POINTER(C.c_double)))
    ne = L.ref_karto_edge_count(h)
    ids, diff, cov = np.zeros((ne, 2), np.int32), np.zeros((ne, 3)), np.zeros((ne, 9))
    if ne:
        L.ref_karto_edges(h, ids.ctypes.data_as(C.POINTER(C.c_int32)), diff.ctypes.data_as(C.POINTER(C.c_double)),
                          cov.ctypes.data_as(C.POINTER(C.c_double)))
    out["edges"] = (ids, diff, cov)
    return out
