"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/libgmapping_ref.so (the reference's real GMapping grid
headers, see oracle/ref_gmapping.cpp)."""
import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/libgmapping_ref.so"
_lib = None


def available():
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        L.refg_map_create.restype = C.c_void_p
        L.refg_map_create.argtypes = [C.c_double] * 7
        L.refg_map_destroy.argtypes = [C.c_void_p]
        L.refg_map_size.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        L.refg_compute_map.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int] + [C.c_double] * 4
        L.refg_copy.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                C.POINTER(C.c_float), C.POINTER(C.c_double)]
        L.refg_grid_line.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32), C.c_int]
        _lib = L
    return _lib


class RefGMap:
    def __init__(self, xmin=-40.0, ymin=-40.0, xmax=40.0, ymax=40.0, delta=0.05):
        self.L = lib()
        self.h = self.L.refg_map_create((xmin + xmax) / 2.0, (ymin + ymax) / 2.0, xmin, ymin, xmax, ymax, delta)
        s = (C.c_int32 * 2)()
        self.L.refg_map_size(self.h, s)
        self.size_x, self.size_y = s[0], s[1]

    def compute_map(self, ranges, angles, laser_xy=(0.0, 0.0), max_range=30 - 0.01, max_urange=25.0):
        r = np.ascontiguousarray(ranges, np.float64)
        a = np.ascontiguousarray(angles, np.float64)
        dp = C.POINTER(C.c_double)
        return self.L.refg_compute_map(self.h, r.ctypes.data_as(dp), a.ctypes.data_as(dp), len(r), laser_xy[0],
                                       laser_xy[1], max_range, max_urange)

    def cells(self):
        c = self.size_x * self.size_y
        n, v = np.zeros(c, np.int32), np.zeros(c, np.int32)
        ax, ay, occ = np.zeros(c, np.float32), np.zeros(c, np.float32), np.zeros(c, np.float64)
        ip, fp = C.POINTER(C.c_int32), C.POINTER(C.c_float)
        self.L.refg_copy(self.h, n.ctypes.data_as(ip), v.ctypes.data_as(ip), ax.ctypes.data_as(fp),
                         ay.ctypes.data_as(fp), occ.ctypes.data_as(C.POINTER(C.c_double)))
        sh = (self.size_y, self.size_x)
        return n.reshape(sh), v.reshape(sh), ax.reshape(sh), ay.reshape(sh), occ.reshape(sh)

    def close(self):
        if self.h:
            self.L.refg_map_destroy(self.h)
            self.h = None


def grid_line(x0, y0, x1, y1):
    cap = abs(x1 - x0) + abs(y1 - y0) + 4
    out = np.zeros((cap, 2), np.int32)
    n = lib().refg_grid_line(x0, y0, x1, y1, out.ctypes.data_as(C.POINTER(C.c_int32)), cap)
    return out[:n].copy()
