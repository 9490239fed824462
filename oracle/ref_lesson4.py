"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson4_ref.so: lesson4's UNMODIFIED make-map nodes,
reference/lesson4/src/gmapping/gmapping.cc and reference/lesson4/src/hector_mapping/hector_mapping.cc, compiled where
they lie against the ROS, message and Eigen stand-ins under oracle/shim/ by
oracle/ref_lesson4_gmapping.cpp and oracle/ref_lesson4_hector.cpp (two translation units: see the latter),
built by oracle/recipes.py from a checkout of the original project; where it is absent the tests replay its
recorded answers (tests/reference_record.py).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/liblesson4_ref.so"
SENTINEL = 0x55  # ref_lesson4_gmapping.cpp: a byte behind the map the node did not write
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        vp = C.c_void_p
        L.ref_l4_clear_params.argtypes = []
        L.ref_l4_clear_params.restype = None
        L.ref_l4_param.argtypes = [C.c_char_p, C.c_double]
        L.ref_l4_param.restype = None
        L.ref_l4_gmapping_new.argtypes = [vp]
        L.ref_l4_gmapping_new.restype = None
        L.ref_l4_gmapping_scan.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
        L.ref_l4_gmapping_slack.argtypes = []
        L.ref_l4_hector_new.argtypes = []
        L.ref_l4_hector_new.restype = None
        L.ref_l4_hector_scan.argtypes = [vp, C.c_int, vp, vp, vp, C.c_long]
        _lib = L
    return _lib


def _params(params: dict):
    L = lib()
    L.ref_l4_clear_params()
    for k, v in params.items():
        L.ref_l4_param(k.encode(), float(v))


def gmapping(params: dict, fields, ranges):
    """A fresh GMapping node with the parameter-server values `params` (the node's names: maxRange, maxUrange, xmin, ymin,
    xmax, ymax, delta, occ_thresh) over one recording.  fields = (angle_min, angle_increment, range_min, range_max)
    float32, ranges [S][n] float32.  -> (maps [k][height][width] int8, k = the scans published before the first the
    node would assert on (S when none), overrun [k][slack] int8: the bytes behind map_.data, SENTINEL where the node
    wrote none, n_overrun [k])."""
    L = lib()
    _params(params)
    dims = np.zeros(2, np.int32)
    L.ref_l4_gmapping_new(dims.ctypes.data)
    w, h = int(dims[0]), int(dims[1])
    slack = L.ref_l4_gmapping_slack()
    f = np.ascontiguousarray(fields, np.float32)
    r = np.ascontiguousarray(ranges, np.float32)
    maps = np.zeros((len(r), h, w), np.int8)
    ov = np.zeros((len(r), slack), np.int8)
    nov = np.zeros(len(r), np.int32)
    for s in range(len(r)):
        n_ov = C.c_int32(0)
        rc = L.ref_l4_gmapping_scan(f.ctypes.data, r.shape[1], r[s].ctypes.data, maps[s].ctypes.data,
                                    ov[s].ctypes.data, slack, C.addressof(n_ov))
        if rc == -1:
            return maps[:s], s, ov[:s], nov[:s]
        assert rc == 0, f"the GMapping node published nothing for scan {s}"
        nov[s] = n_ov.value
    return maps, len(r), ov, nov


def hector(params: dict, fields, ranges) -> np.ndarray:
    """A fresh Hector make-map node with the parameter-server values `params` (xmin, ymin, xmax, ymax, delta) over one
    recording (arguments as for gmapping) -> maps [S][height][width] int8."""
    L = lib()
    _params(params)
    L.ref_l4_hector_new()
    f = np.ascontiguousarray(fields, np.float32)
    r = np.ascontiguousarray(ranges, np.float32)
    out, info = None, np.zeros(2, np.int32)
    for s in range(len(r)):
        buf = np.zeros(1 << 24, np.int8) if out is None else out[s]
        rc = L.ref_l4_hector_scan(f.ctypes.data, r.shape[1], r[s].ctypes.data, info.ctypes.data, buf.ctypes.data,
                                  buf.size)
        if rc == -3 and out is None:  # a map larger than the first buffer: its size is known now, and a scan's map is
            buf = np.zeros(int(info[0]) * int(info[1]), np.int8)  # fresh, so the scan can run again
            rc = L.ref_l4_hector_scan(f.ctypes.data, r.shape[1], r[s].ctypes.data, info.ctypes.data, buf.ctypes.data,
                                      buf.size)
        assert rc == 0, f"the Hector node published nothing for scan {s} ({rc})"
        if out is None:
            out = np.zeros((len(r), info[1], info[0]), np.int8)
            out[0] = buf[:info[0] * info[1]].reshape(info[1], info[0])
    return out if out is not None else np.zeros((0, 0, 0), np.int8)
