"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/libkarto_ref*.so (the UNMODIFIED reference
open_karto compiled by oracle/recipes.py).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes


class MatcherParams(C.Structure):
    """Mirror of ref_matcher_params (oracle/ref_driver.cpp).  Defaults = Mapper.cpp:1569-1652."""
    _fields_ = [("search_size", C.c_double), ("resolution", C.c_double), ("smear_deviation", C.c_double),
                ("range_threshold", C.c_double), ("distance_variance_penalty", C.c_double),
                ("angle_variance_penalty", C.c_double), ("fine_search_angle_offset", C.c_double),
                ("coarse_search_angle_offset", C.c_double), ("coarse_angle_resolution", C.c_double),
                ("minimum_angle_penalty", C.c_double), ("minimum_distance_penalty", C.c_double),
                ("use_response_expansion", C.c_int32), ("_pad", C.c_int32)]


class LaserParams(C.Structure):
    _fields_ = [("type", C.c_int32), ("_pad", C.c_int32), ("min_angle", C.c_double), ("max_angle", C.c_double),
                ("angular_resolution", C.c_double), ("min_range", C.c_double), ("max_range", C.c_double),
                ("range_threshold", C.c_double), ("offset_pose", C.c_double * 3)]


KT_PI_180 = 0.01745329251994329577


def default_matcher_params(search_size=0.3, resolution=0.01, smear=0.03, range_threshold=12.0, **kw) -> MatcherParams:
    p = MatcherParams(search_size, resolution, smear, range_threshold,
                      0.3 * 0.3, (20 * KT_PI_180) ** 2, 0.2 * KT_PI_180, 20 * KT_PI_180, 2 * KT_PI_180,
                      0.9, 0.5, 0, 0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def laser_params(laser) -> LaserParams:
    return LaserParams(laser.type, 0, laser.min_angle, laser.max_angle, laser.angular_resolution, laser.min_range,
                       laser.max_range, laser.range_threshold, (C.c_double * 3)(*laser.offset_pose))


def _name(ndebug: bool) -> str:
    return "_ref/libkarto_ref_ndebug.so" if ndebug else "_ref/libkarto_ref.so"


def available(ndebug: bool = False) -> bool:
    return recipes.available(_name(ndebug))


_libs = {}


def _lib(ndebug: bool):
    if ndebug in _libs:
        return _libs[ndebug]
    L = C.CDLL(recipes.path(_name(ndebug)))
    dp, ip, u8p, u32p = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
    L.ref_session_create.restype = C.c_void_p
    L.ref_session_create.argtypes = [C.POINTER(MatcherParams), C.POINTER(LaserParams)]
    L.ref_session_destroy.argtypes = [C.c_void_p]
    L.ref_n_readings.argtypes = [C.c_void_p]
    L.ref_laser_validate.argtypes = [C.c_void_p]
    L.ref_scan_add.argtypes = [C.c_void_p, dp, C.c_int, dp]
    L.ref_scan_set_pose.argtypes = [C.c_void_p, C.c_int, dp]
    L.ref_scan_sensor_pose.argtypes = [C.c_void_p, C.c_int, dp]
    L.ref_scan_point_readings.argtypes = [C.c_void_p, C.c_int, C.c_int, dp, C.c_int]
    L.ref_find_valid_points.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_int]
    L.ref_grid_info.argtypes = [C.c_void_p, ip, dp]
    L.ref_grid_copy.argtypes = [C.c_void_p, u8p]
    L.ref_kernel_copy.argtypes = [C.c_void_p, u8p]
    L.ref_set_grid_from_scans.argtypes = [C.c_void_p, C.c_int, ip, C.c_int]
    L.ref_match_scan.argtypes = [C.c_void_p, C.c_int, ip, C.c_int, C.c_int, C.c_int, dp, dp, dp]
    L.ref_correlate_scan.argtypes = [C.c_void_p, C.c_int, dp] + [C.c_double] * 6 + [C.c_int, C.c_int, dp, dp, dp]
    L.ref_compute_offsets.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, ip, C.c_int]
    L.ref_response_sums.argtypes = [C.c_void_p, C.c_int, dp] + [C.c_double] * 6 + [ip, C.c_int, ip]
    L.ref_time_correlate.restype = C.c_double
    L.ref_time_correlate.argtypes = [C.c_void_p, C.c_int, dp] + [C.c_double] * 6 + [C.c_int, C.c_int, C.c_int, dp]
    L.ref_time_match_scan.restype = C.c_double
    L.ref_time_match_scan.argtypes = [C.c_void_p, C.c_int, ip, C.c_int, C.c_int, dp]
    L.ref_occgrid_create.restype = C.c_void_p
    L.ref_occgrid_create.argtypes = [C.c_void_p, ip, C.c_int, C.c_double, ip, dp]
    L.ref_occgrid_copy.argtypes = [C.c_void_p, u8p, u32p, u32p]
    L.ref_occgrid_destroy.argtypes = [C.c_void_p]
    L.ref_time_occgrid.restype = C.c_double
    L.ref_time_occgrid.argtypes = [C.c_void_p, ip, C.c_int, C.c_double, C.c_int, dp]
    L.ref_trace_line.argtypes = [C.c_int] * 6 + [ip, C.c_int]
    _libs[ndebug] = L
    return L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


class RefSession:
    """One reference ScanMatcher + one registered LaserRangeFinder + a list of LocalizedRangeScans."""

    def __init__(self, params: MatcherParams, laser, ndebug: bool = False):
        self.L = _lib(ndebug)
        self.params = params
        lp = laser_params(laser)
        self.h = self.L.ref_session_create(C.byref(params), C.byref(lp))
        if not self.h:
            raise ValueError("ScanMatcher::Create returned NULL (bad parameters)")
        self.n_readings = self.L.ref_n_readings(self.h)

    def close(self):
        if self.h:
            self.L.ref_session_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def laser_validate(self) -> int:
        self.n_readings = self.L.ref_laser_validate(self.h)
        return self.n_readings

    def add_scan(self, ranges, pose) -> int:
        r = np.ascontiguousarray(ranges, dtype=np.float64)
        p = np.ascontiguousarray(pose, dtype=np.float64)
        return self.L.ref_scan_add(self.h, _dp(r), len(r), _dp(p))

    def set_pose(self, scan, pose):
        p = np.ascontiguousarray(pose, dtype=np.float64)
        self.L.ref_scan_set_pose(self.h, scan, _dp(p))

    def sensor_pose(self, scan):
        out = np.zeros(3)
        self.L.ref_scan_sensor_pose(self.h, scan, _dp(out))
        return out

    def point_readings(self, scan, filtered=False):
        out = np.zeros((self.n_readings + 8, 2))
        n = self.L.ref_scan_point_readings(self.h, scan, int(filtered), _dp(out), len(out))
        return out[:n].copy()

    def find_valid_points(self, scan, viewpoint):
        out = np.zeros((self.n_readings + 8, 2))
        vp = np.ascontiguousarray(viewpoint, dtype=np.float64)
        n = self.L.ref_find_valid_points(self.h, scan, _dp(vp), _dp(out), len(out))
        return out[:n].copy()

    def grid_info(self):
        info = np.zeros(9, dtype=np.int32)
        off = np.zeros(2)
        self.L.ref_grid_info(self.h, _ip(info), _dp(off))
        keys = ["width", "height", "width_step", "data_size", "roi_x", "roi_y", "roi_w", "roi_h", "kernel_size"]
        d = {k: int(v) for k, v in zip(keys, info)}
        d["offset"] = off
        return d

    def grid(self):
        gi = self.grid_info()
        out = np.zeros(gi["data_size"], dtype=np.uint8)
        self.L.ref_grid_copy(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out

    def kernel(self):
        k = self.grid_info()["kernel_size"]
        out = np.zeros(k * k, dtype=np.uint8)
        self.L.ref_kernel_copy(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out.reshape(k, k)

    def set_grid_from_scans(self, scan, base):
        b = np.ascontiguousarray(base, dtype=np.int32)
        rc = self.L.ref_set_grid_from_scans(self.h, scan, _ip(b), len(b))
        if rc:
            raise RuntimeError("reference threw in AddScans")

    def match_scan(self, scan, base, do_penalize=True, do_refine=True):
        b = np.ascontiguousarray(base, dtype=np.int32)
        resp = C.c_double(0)
        mean, cov = np.zeros(3), np.zeros(9)
        rc = self.L.ref_match_scan(self.h, scan, _ip(b), len(b), int(do_penalize), int(do_refine), C.byref(resp),
                                   _dp(mean), _dp(cov))
        if rc:
            raise RuntimeError("reference threw in MatchScan")
        return resp.value, mean, cov.reshape(3, 3)

    def correlate_scan(self, scan, center, off_xy, res_xy, off_a, res_a, do_penalize=True, fine=False, cov_in=None):
        c = np.ascontiguousarray(center, dtype=np.float64)
        resp = C.c_double(0)
        mean = np.zeros(3)
        cov = np.zeros(9) if cov_in is None else np.ascontiguousarray(cov_in, dtype=np.float64).reshape(9).copy()
        rc = self.L.ref_correlate_scan(self.h, scan, _dp(c), off_xy[0], off_xy[1], res_xy[0], res_xy[1], off_a, res_a,
                                       int(do_penalize), int(fine), C.byref(resp), _dp(mean), _dp(cov))
        if rc:
            raise RuntimeError("reference threw in CorrelateScan")
        return resp.value, mean, cov.reshape(3, 3)

    def compute_offsets(self, scan, angle_center, angle_offset, angle_res):
        n_angles = int(_karto_round(angle_offset * 2.0 / angle_res) + 1)
        out = np.zeros(n_angles * self.n_readings, dtype=np.int32)
        na = self.L.ref_compute_offsets(self.h, scan, angle_center, angle_offset, angle_res, _ip(out), len(out))
        assert na == n_angles
        return out.reshape(n_angles, self.n_readings)

    def response_sums(self, scan, center, off_xy, res_xy, off_a, res_a):
        """int32 [nY, nX, nAngles] numerators of GetResponse over the CorrelateScan sweep."""
        c = np.ascontiguousarray(center, dtype=np.float64)
        nx = int(_karto_round(off_xy[0] * 2.0 / res_xy[0]) + 1)
        ny = int(_karto_round(off_xy[1] * 2.0 / res_xy[1]) + 1)
        na = int(_karto_round(off_a * 2.0 / res_a) + 1)
        out = np.zeros(nx * ny * na, dtype=np.int32)
        dims = np.zeros(3, dtype=np.int32)
        rc = self.L.ref_response_sums(self.h, scan, _dp(c), off_xy[0], off_xy[1], res_xy[0], res_xy[1], off_a, res_a,
                                      _ip(out), len(out), _ip(dims))
        if rc:
            raise RuntimeError("reference threw in response sweep")
        assert tuple(dims) == (ny, nx, na)
        return out.reshape(ny, nx, na)

    def time_correlate(self, scan, center, off_xy, res_xy, off_a, res_a, do_penalize=True, fine=False, reps=5):
        c = np.ascontiguousarray(center, dtype=np.float64)
        secs = np.zeros(reps)
        self.L.ref_time_correlate(self.h, scan, _dp(c), off_xy[0], off_xy[1], res_xy[0], res_xy[1], off_a, res_a,
                                  int(do_penalize), int(fine), reps, _dp(secs))
        return secs

    def time_match_scan(self, scan, base, reps=5):
        b = np.ascontiguousarray(base, dtype=np.int32)
        secs = np.zeros(reps)
        self.L.ref_time_match_scan(self.h, scan, _ip(b), len(b), reps, _dp(secs))
        return secs

    def occupancy_grid(self, scans, resolution):
        """-> dict(width,height,width_step,offset,cells u8[h,step],pass u32[h,step],hit u32[h,step]) or None"""
        s = np.ascontiguousarray(scans, dtype=np.int32)
        dims = np.zeros(3, dtype=np.int32)
        off = np.zeros(2)
        g = self.L.ref_occgrid_create(self.h, _ip(s), len(s), resolution, _ip(dims), _dp(off))
        if not g:
            return None
        w, h, step = (int(x) for x in dims)
        cells = np.zeros(step * h, dtype=np.uint8)
        pas = np.zeros(step * h, dtype=np.uint32)
        hit = np.zeros(step * h, dtype=np.uint32)
        self.L.ref_occgrid_copy(g, cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                pas.ctypes.data_as(C.POINTER(C.c_uint32)), hit.ctypes.data_as(C.POINTER(C.c_uint32)))
        self.L.ref_occgrid_destroy(g)
        return dict(width=w, height=h, width_step=step, offset=off, cells=cells.reshape(h, step),
                    passes=pas.reshape(h, step), hits=hit.reshape(h, step))

    def time_occgrid(self, scans, resolution, reps=5):
        s = np.ascontiguousarray(scans, dtype=np.int32)
        secs = np.zeros(reps)
        self.L.ref_time_occgrid(self.h, _ip(s), len(s), resolution, reps, _dp(secs))
        return secs


def trace_line(w, h, x0, y0, x1, y1, ndebug=False):
    cap = 2 * (abs(x1 - x0) + abs(y1 - y0) + 4)
    out = np.zeros((cap, 2), dtype=np.int32)
    n = _lib(ndebug).ref_trace_line(w, h, x0, y0, x1, y1, _ip(out), cap)
    return out[:n].copy()


def _karto_round(v: float) -> float:
    """math::Round (Math.h:87-90)."""
    import math
    return math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5)


# ---------------------------------------------------------------- the whole front end: karto::Mapper::Process

class RefMapper:
    """karto::Mapper (Mapper.cpp:1999-2079) fed one LaserScan at a time, as karto_slam.cc:437-475 does.  `params` is a
    creating-..._b200.mapper.MapperParams (ref_mapper_params has the same layout); `laser` a synth.Laser."""

    def __init__(self, params, laser, ndebug: bool = False):
        self.L = _lib(ndebug)
        self.L.ref_mapper_create.restype = C.c_void_p
        self.lp = laser_params(laser)
        self.h = C.c_void_p(self.L.ref_mapper_create(C.byref(params), C.byref(self.lp)))
        self.n = laser.n_readings
        self._keep = []

    def set_scan_solver(self, solver):
        """solver: any ctypes struct laid out as b2s_scan_solver / ref_scan_solver."""
        self._keep.append(solver)
        self.L.ref_mapper_set_solver(self.h, C.byref(solver))

    def add_sensor(self, prefix: str) -> int:
        """Another robot's laser (same parameters); its name is `prefix`_<n>, the session's own is ref_mapper_laser_<n>
        (the order of the names decides the order sensors are visited in, Karto.h:484).  Returns the sensor index."""
        return int(self.L.ref_mapper_add_sensor(self.h, prefix.encode()))

    def process(self, ranges, odometric_pose, time=0.0, sensor=0):
        r, o, out = np.ascontiguousarray(ranges, np.float64), np.ascontiguousarray(odometric_pose, np.float64), np.zeros(3)
        if sensor == 0:
            ok = self.L.ref_mapper_process(self.h, _dp(r), self.n, _dp(o), C.c_double(time), _dp(out))
        else:
            ok = self.L.ref_mapper_process_sensor(self.h, int(sensor), _dp(r), self.n, _dp(o), C.c_double(time), _dp(out))
        return bool(ok), out

    def poses_by_id(self):
        out = np.zeros((self.L.ref_mapper_scan_count(self.h), 3))
        if len(out):
            self.L.ref_mapper_get_poses_by_id(self.h, _dp(out))
        return out

    def poses(self):
        out = np.zeros((self.L.ref_mapper_scan_count(self.h), 3))
        if len(out):
            self.L.ref_mapper_get_poses(self.h, _dp(out))
        return out

    def edges(self):
        n = self.L.ref_mapper_edge_count(self.h)
        ids, diff, cov = np.zeros((n, 2), np.int32), np.zeros((n, 3)), np.zeros((n, 9))
        if n:
            self.L.ref_mapper_get_edges(self.h, _ip(ids), _dp(diff), _dp(cov))
        return ids, diff, cov.reshape(n, 3, 3)

    def running_count(self):
        return self.L.ref_mapper_running_count(self.h)

    def close(self):
        if self.h:
            self.L.ref_mapper_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
