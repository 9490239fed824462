"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/libhector_ref.so: the UNMODIFIED lesson4 Hector headers
(GridMap, OccGridMapUtil, ScanMatcher, HectorSlamProcessor) compiled by oracle/recipes.py against the Eigen stand-in
oracle/shim/Eigen/mini_eigen.h.  RefHectorMap has the interface of oracle.port.PortHectorMap.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/libhector_ref.so"
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        L.ref_hmap_create.restype = C.c_void_p
        L.ref_hmap_update_by_scan.restype = C.c_long
        L.ref_hmap_update_by_scan_just_once.restype = C.c_long
        L.ref_hproc_create.restype = C.c_void_p
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, np.float32)
    return a.reshape(shape) if shape else a


class RefHectorMap:
    """One hectorslam::GridMap + its OccGridMapUtil + ScanMatcher (one level of MapRepMultiMap)."""

    def __init__(self, size_x, size_y, resolution, start_x=0.5, start_y=0.5):
        self.L = lib()
        self.sx, self.sy = size_x, size_y
        self.h = C.c_void_p(self.L.ref_hmap_create(size_x, size_y, C.c_float(resolution), C.c_float(start_x),
                                                   C.c_float(start_y)))

    def set_factors(self, update_free, update_occupied):
        self.L.ref_hmap_set_factors(self.h, C.c_float(update_free), C.c_float(update_occupied))

    def update_by_scan(self, points, origo, world_pose):
        p, o, w = _f32(points, (-1, 2)), _f32(origo), _f32(world_pose)
        return self.L.ref_hmap_update_by_scan(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float), _p(w, C.c_float))

    def update_by_scan_just_once(self, points_m, origo):
        p, o = _f32(points_m, (-1, 2)), _f32(origo)
        return self.L.ref_hmap_update_by_scan_just_once(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float))

    def match_data(self, points, begin_world_pose, max_iterations):
        p, b = _f32(points, (-1, 2)), _f32(begin_world_pose)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self.L.ref_hmap_match_data(self.h, _p(p, C.c_float), len(p), _p(b, C.c_float), max_iterations,
                                   _p(pose, C.c_float), _p(cov, C.c_float))
        return pose, cov.reshape(3, 3)

    def cells(self):
        lo, ui = np.zeros(self.sx * self.sy, np.float32), np.zeros(self.sx * self.sy, np.int32)
        self.L.ref_hmap_copy(self.h, _p(lo, C.c_float), _p(ui, C.c_int32))
        return lo.reshape(self.sy, self.sx), ui.reshape(self.sy, self.sx)

    def close(self):
        if self.h:
            self.L.ref_hmap_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def line_cells(size, x0, y0, x1, y1):
    """Cells OccGridMapBase::updateLineBresenhami frees / occupies for one beam on a scratch size x size map."""
    free = np.zeros(4 * size, np.int32)
    nf, occ = C.c_int32(0), C.c_int32(-1)
    lib().ref_hector_line_cells(size, x0, y0, x1, y1, _p(free, C.c_int32), C.byref(nf), C.byref(occ))
    return free[:nf.value].copy(), occ.value


class RefHectorProcessor:
    """hectorslam::HectorSlamProcessor (HectorSlamProcessor.h): multi-level matchData + updateByScan."""

    def __init__(self, resolution=0.05, size_x=1024, size_y=1024, start=(0.5, 0.5), levels=3,
                 update_free=0.4, update_occupied=0.9, min_dist=0.4, min_angle=0.13):
        self.L = lib()
        self.levels = levels
        self.h = C.c_void_p(self.L.ref_hproc_create(C.c_float(resolution), size_x, size_y, C.c_float(start[0]),
                                                    C.c_float(start[1]), levels, C.c_float(update_free),
                                                    C.c_float(update_occupied), C.c_float(min_dist), C.c_float(min_angle)))

    def update(self, points, origo, pose_hint, map_without_matching=False):
        p, o, w = _f32(points, (-1, 2)), _f32(origo), _f32(pose_hint)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self.L.ref_hproc_update(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float), _p(w, C.c_float),
                                int(map_without_matching), _p(pose, C.c_float), _p(cov, C.c_float))
        return pose, cov.reshape(3, 3)

    def level(self, i):
        dims = (C.c_int * 2)()
        assert self.L.ref_hproc_level_dims(self.h, i, dims) == 0
        sx, sy = dims[0], dims[1]
        lo, ui = np.zeros(sx * sy, np.float32), np.zeros(sx * sy, np.int32)
        self.L.ref_hproc_copy_level(self.h, i, _p(lo, C.c_float), _p(ui, C.c_int32))
        return lo.reshape(sy, sx), ui.reshape(sy, sx)

    def close(self):
        if self.h:
            self.L.ref_hproc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
