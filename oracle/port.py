"""TEST INFRASTRUCTURE — ctypes binding of oracle/libslam_oracle.so, the plain-C CPU restatement
(karto_oracle.c / gmapping_oracle.c / hector_oracle.c).  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module; the product never does.
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
        L = C.CDLL(recipes.build("libslam_oracle.so"))
        L.orc_round.restype = C.c_double
        L.orc_round.argtypes = [C.c_double]
        L.orc_normalize_angle.restype = C.c_double
        L.orc_normalize_angle.argtypes = [C.c_double]
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _d(a):
    return _p(a, C.c_double)


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class PortMatcher:
    """Stateful convenience wrapper with the same call sequence as the product handle / RefSession."""

    def __init__(self, params, laser):
        self.L = lib()
        self.p = params
        self.l = laser
        self.g = abi.GridInfo()
        rc = self.L.orc_matcher_layout(C.byref(params), C.byref(self.g))
        if rc:
            raise ValueError(f"orc_matcher_layout -> {abi.STATUS_NAMES[rc]}")
        self.n = laser.n_readings
        self.grid = np.zeros(self.g.data_size, dtype=np.uint8)
        self.grid_off = np.zeros(2)
        self.last_sums = None

    def kernel(self):
        k = self.g.kernel_size
        K = np.zeros(k * k, dtype=np.uint8)
        self.L.orc_smear_kernel(C.c_double(self.p.resolution), C.c_double(self.p.smear_deviation), k, _p(K, C.c_uint8))
        return K.reshape(k, k)

    def sensor_pose(self, robot_pose):
        out = np.zeros(3)
        off = f64(list(self.l.offset_pose))
        self.L.orc_sensor_pose(_d(f64(robot_pose)), _d(off), _d(out))
        return out

    def point_readings(self, ranges, robot_pose):
        out = np.zeros((self.n, 2))
        self.L.orc_point_readings(C.byref(self.l), _d(f64(ranges)), _d(f64(robot_pose)), _d(out))
        return out

    def find_valid_points(self, pts, viewpoint):
        pts = f64(pts)
        out = np.zeros_like(pts)
        n = self.L.orc_find_valid_points(_d(pts), len(pts), _d(f64(viewpoint)), _d(out))
        return out[:n].copy()

    def set_scan(self, ranges, robot_pose):
        self.ranges = f64(ranges)
        self.robot_pose = f64(robot_pose)
        self.sp = self.sensor_pose(robot_pose)
        self.pts = self.point_readings(ranges, robot_pose)

    def add_scans(self, base_ranges, base_poses):
        br, bp = f64(base_ranges).reshape(-1, self.n), f64(base_poses).reshape(-1, 3)
        self.L.orc_grid_offset(C.byref(self.g), C.c_double(self.p.resolution), _d(self.sp), _d(self.grid_off))
        self.L.orc_add_scans(C.byref(self.p), C.byref(self.l), C.byref(self.g), _d(self.grid_off),
                             _p(self.grid, C.c_uint8), len(br), _d(br), _d(bp), _d(self.sp[:2].copy()))

    def compute_offsets(self, angle_center, angle_offset, angle_res):
        na = abi.n_steps(angle_offset, angle_res)
        lut = np.zeros((na, self.n), dtype=np.int32)
        self.L.orc_compute_offsets(C.byref(self.g), C.c_double(self.p.resolution), _d(self.grid_off), _d(self.ranges),
                                   _d(self.pts), self.n, _d(self.sp), C.c_double(angle_center),
                                   C.c_double(angle_offset), C.c_double(angle_res), _p(lut, C.c_int32))
        return lut

    def correlate_scan(self, center, search, cov_in=None, want_sums=False):
        res = abi.MatchResult()
        if cov_in is not None:
            for i, v in enumerate(np.asarray(cov_in, dtype=np.float64).reshape(9)):
                res.cov[i] = v
        nx, ny = abi.n_steps(search.offset_x, search.res_x), abi.n_steps(search.offset_y, search.res_y)
        na = abi.n_steps(search.angle_offset, search.angle_res)
        sums = np.zeros((ny, nx, na), dtype=np.int32) if want_sums else None
        rc = self.L.orc_correlate_scan(C.byref(self.p), C.byref(self.g), _d(self.grid_off), _p(self.grid, C.c_uint8),
                                       _d(self.ranges), _d(self.pts), self.n, _d(self.sp), _d(f64(center)),
                                       C.byref(search), C.byref(res), _p(sums, C.c_int32) if want_sums else None)
        self.last_sums = sums
        return rc, res

    def match_scan(self, ranges, robot_pose, base_ranges, base_poses, do_penalize=True, do_refine=True):
        br, bp = f64(base_ranges).reshape(-1, self.n), f64(base_poses).reshape(-1, 3)
        res = abi.MatchResult()
        rc = self.L.orc_match_scan(C.byref(self.p), C.byref(self.l), _d(f64(ranges)), _d(f64(robot_pose)), len(br),
                                   _d(br), _d(bp), int(do_penalize), int(do_refine), C.byref(res),
                                   _p(self.grid, C.c_uint8), _d(self.grid_off))
        return rc, res


def occupancy_grid(laser, ranges, poses, resolution):
    L = lib()
    r, p = f64(ranges).reshape(-1, laser.n_readings), f64(poses).reshape(-1, 3)
    info = abi.OccGridInfo()
    L.orc_occ_dimensions(C.byref(laser), len(r), _d(r), _d(p), C.c_double(resolution), C.byref(info))
    n = info.data_size
    pas, hit, cells = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8)
    L.orc_occ_create_from_scans(C.byref(laser), len(r), _d(r), _d(p), C.byref(info), _p(pas, C.c_uint32),
                                _p(hit, C.c_uint32), _p(cells, C.c_uint8))
    h, s = info.height, info.width_step
    return dict(width=info.width, height=h, width_step=s, offset=np.array(info.offset[:]),
                cell_visits=int(info.cell_visits), cells=cells.reshape(h, s), passes=pas.reshape(h, s),
                hits=hit.reshape(h, s))


def trace_line(w, h, x0, y0, x1, y1):
    cap = abs(x1 - x0) + abs(y1 - y0) + 4
    out = np.zeros((cap, 2), dtype=np.int32)
    n = lib().orc_trace_line_cells(w, h, x0, y0, x1, y1, _p(out, C.c_int32), cap)
    return out[:n].copy()


def result_tuple(res):
    return res.response, np.array(res.pose[:]), np.array(res.cov[:]).reshape(3, 3)


# ---------------------------------------------------------------- GMapping (gmapping_oracle.c)

class PortGMap:
    def __init__(self, xmin=-40.0, ymin=-40.0, xmax=40.0, ymax=40.0, delta=0.05):
        self.L = lib()
        self.bounds = (xmin, ymin, xmax, ymax, delta)
        self.cx, self.cy = (xmin + xmax) / 2.0, (ymin + ymax) / 2.0
        self.layout = np.zeros(4, np.int32)
        self.L.orc_gmap_layout(C.c_double(self.cx), C.c_double(self.cy), C.c_double(xmin), C.c_double(ymin),
                               C.c_double(xmax), C.c_double(ymax), C.c_double(delta), _p(self.layout, C.c_int32))
        self.size_x, self.size_y = int(self.layout[0]), int(self.layout[1])
        c = self.size_x * self.size_y
        self.n, self.visits = np.zeros(c, np.int32), np.zeros(c, np.int32)
        self.acc_x, self.acc_y = np.zeros(c, np.float32), np.zeros(c, np.float32)

    def compute_map(self, ranges, angles, laser_xy=(0.0, 0.0), max_range=30 - 0.01, max_urange=25.0):
        r, a = f64(ranges), f64(angles)
        return self.L.orc_gmap_compute_map(C.c_double(self.cx), C.c_double(self.cy), C.c_double(self.bounds[4]),
                                           _p(self.layout, C.c_int32), _d(r), _d(a), len(r), C.c_double(laser_xy[0]),
                                           C.c_double(laser_xy[1]), C.c_double(max_range), C.c_double(max_urange),
                                           _p(self.n, C.c_int32), _p(self.visits, C.c_int32), _p(self.acc_x, C.c_float),
                                           _p(self.acc_y, C.c_float))

    def cells(self):
        sh = (self.size_y, self.size_x)
        return self.n.reshape(sh), self.visits.reshape(sh), self.acc_x.reshape(sh), self.acc_y.reshape(sh)

    def ros_map(self, occ_thresh=0.25):
        xmin, ymin, xmax, ymax, delta = self.bounds
        w, h = int((xmax - xmin) / delta), int((ymax - ymin) / delta)
        out = np.zeros((h, w), np.int8)
        self.L.orc_gmap_ros(_p(self.layout, C.c_int32), _p(self.n, C.c_int32), _p(self.visits, C.c_int32),
                            C.c_double(occ_thresh), w, h, _p(out, C.c_int8))
        return out


def gmap_grid_line(x0, y0, x1, y1):
    cap = abs(x1 - x0) + abs(y1 - y0) + 4
    out = np.zeros((cap, 2), np.int32)
    n = lib().orc_gmap_grid_line(x0, y0, x1, y1, _p(out, C.c_int32), cap)
    return out[:n].copy()


def mapper_match_hook(mapper_params, laser):
    """A b2s_match_scan_fn (include/b200slam.h) served by the CPU restatement's MatchScan — TESTS ONLY: it lets the
    host-side graph logic of the product's mapper (karto_mapper.cu) run on a machine without a GPU.  Returns a Python
    callable for creating-..._b200.mapper.Mapper(match_fn=...)."""
    L = lib()
    n = laser.n_readings
    matchers = [PortMatcher(mapper_params.sequential, laser), PortMatcher(mapper_params.loop, laser)]

    def hook(user, which, batch, ranges, poses, base_first, n_base, base_ranges, base_poses, do_penalize, do_refine, results):
        pm = matchers[which]
        for b in range(batch):
            r = np.ctypeslib.as_array(ranges, shape=((b + 1) * n,))[b * n:(b + 1) * n]
            p = np.ctypeslib.as_array(poses, shape=((b + 1) * 3,))[b * 3:(b + 1) * 3]
            f, c = base_first[b], n_base[b]
            br = np.ctypeslib.as_array(base_ranges, shape=((f + c) * n,))[f * n:(f + c) * n]
            bp = np.ctypeslib.as_array(base_poses, shape=((f + c) * 3,))[f * 3:(f + c) * 3]
            rc, res = pm.match_scan(r, p, br, bp, bool(do_penalize), bool(do_refine))
            if rc:
                return rc
            C.memmove(C.byref(results[b]), C.byref(res), C.sizeof(res))
        return 0

    return hook


# ---------------------------------------------------------------- Hector (hector_oracle.c) — pinned against
# oracle/ref_hector.cpp (the reference headers compiled with the Eigen stand-in) by tests/test_oracle_hector_reference.py

class PortHectorMap:
    def __init__(self, size_x, size_y, resolution, start_x=0.5, start_y=0.5):
        self.L = lib()
        self.L.orc_hmap_create.restype = C.c_void_p
        self.L.orc_hmap_update_by_scan.restype = C.c_long
        self.sx, self.sy = size_x, size_y
        self.h = C.c_void_p(self.L.orc_hmap_create(size_x, size_y, C.c_float(resolution), C.c_float(start_x),
                                                   C.c_float(start_y)))

    def set_factors(self, update_free, update_occupied):
        self.L.orc_hmap_set_factors(self.h, C.c_float(update_free), C.c_float(update_occupied))

    def update_by_scan(self, points, origo, world_pose):
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 2)
        o, w = np.ascontiguousarray(origo, np.float32), np.ascontiguousarray(world_pose, np.float32)
        return self.L.orc_hmap_update_by_scan(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float), _p(w, C.c_float))

    def update_by_scan_just_once(self, points_m, origo):
        p = np.ascontiguousarray(points_m, np.float32).reshape(-1, 2)
        o = np.ascontiguousarray(origo, np.float32)
        self.L.orc_hmap_update_by_scan_just_once.restype = C.c_long
        return self.L.orc_hmap_update_by_scan_just_once(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float))

    def match_data(self, points, begin_world_pose, max_iterations):
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 2)
        b = np.ascontiguousarray(begin_world_pose, np.float32)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self.L.orc_hmap_match_data(self.h, _p(p, C.c_float), len(p), _p(b, C.c_float), max_iterations,
                                   _p(pose, C.c_float), _p(cov, C.c_float))
        return pose, cov.reshape(3, 3)

    def cells(self):
        lo, ui = np.zeros(self.sx * self.sy, np.float32), np.zeros(self.sx * self.sy, np.int32)
        self.L.orc_hmap_copy(self.h, _p(lo, C.c_float), _p(ui, C.c_int32))
        return lo.reshape(self.sy, self.sx), ui.reshape(self.sy, self.sx)

    def close(self):
        if self.h:
            self.L.orc_hmap_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PortHectorProcessor:
    """orc_hproc_* — HectorSlamProcessor / MapRepMultiMap restatement; interface of oracle.ref_hector.RefHectorProcessor."""

    def __init__(self, resolution=0.05, size_x=1024, size_y=1024, start=(0.5, 0.5), levels=3,
                 update_free=0.4, update_occupied=0.9, min_dist=0.4, min_angle=0.13):
        self.L = lib()
        self.L.orc_hproc_create.restype = C.c_void_p
        self.levels = levels
        self.h = C.c_void_p(self.L.orc_hproc_create(C.c_float(resolution), size_x, size_y, C.c_float(start[0]),
                                                    C.c_float(start[1]), levels))
        self.L.orc_hproc_set_params(self.h, C.c_float(update_free), C.c_float(update_occupied), C.c_float(min_dist),
                                    C.c_float(min_angle))

    def update(self, points, origo, pose_hint, map_without_matching=False):
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 2)
        o, w = np.ascontiguousarray(origo, np.float32), np.ascontiguousarray(pose_hint, np.float32)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self.L.orc_hproc_update(self.h, _p(p, C.c_float), len(p), _p(o, C.c_float), _p(w, C.c_float),
                                int(map_without_matching), _p(pose, C.c_float), _p(cov, C.c_float))
        self.map_updated = bool(self.L.orc_hproc_map_updated(self.h))  # the gate's decision, as HectorSlam reports it
        return pose, cov.reshape(3, 3)

    def level(self, i):
        dims = (C.c_int * 2)()
        assert self.L.orc_hproc_level_dims(self.h, i, dims) == 0
        sx, sy = dims[0], dims[1]
        lo, ui = np.zeros(sx * sy, np.float32), np.zeros(sx * sy, np.int32)
        self.L.orc_hproc_copy_level(self.h, i, _p(lo, C.c_float), _p(ui, C.c_int32))
        return lo.reshape(sy, sx), ui.reshape(sy, sx)

    def close(self):
        if self.h:
            self.L.orc_hproc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---------------------------------------------------------------- PL-ICP (plicp_oracle.c) — PARITY UNPINNED

def plicp_match(params, ref_ranges, sens_ranges, theta, range_min, range_max, first_guess):
    r, s_, t = f64(ref_ranges), f64(sens_ranges), f64(theta)
    res = abi.IcpResult()
    lib().orc_plicp_match(C.byref(params), len(t), _d(r), _d(s_), _d(t), C.c_double(range_min), C.c_double(range_max),
                          _d(f64(first_guess)), C.byref(res))
    return res


# ---------------------------------------------------------------- lesson5 de-skew (deskew_oracle.c) — pinned except PCL / Eigen

def deskew_integrate_imu(stamps, angular_velocity, scan_start, scan_end, capacity=2000):
    L = lib()
    dp = C.POINTER(C.c_double)
    L.orc_deskew_integrate_imu.argtypes = [C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, dp, dp, dp, dp]
    L.orc_deskew_integrate_imu.restype = C.c_int32
    st, av = f64(stamps), f64(angular_velocity).reshape(-1, 3)
    t, x, y, z = (np.zeros(capacity) for _ in range(4))
    last = L.orc_deskew_integrate_imu(len(st), _d(st), _d(av), float(scan_start), float(scan_end), capacity, _d(t), _d(x), _d(y), _d(z))
    return int(last), t, x, y, z


def deskew_odom_increment(start_pose, end_pose):
    L = lib()
    out = np.zeros(3, np.float32)
    L.orc_deskew_odom_increment.restype = None
    L.orc_deskew_odom_increment(_d(f64(start_pose)), _d(f64(end_pose)), out.ctypes.data_as(C.POINTER(C.c_float)))
    return out


def deskew_scan(ranges, angle_min, angle_increment, info, imu_time, rot_x, rot_y, rot_z):
    """info: any ctypes struct laid out as b2s_deskew_scan.  -> corrected cloud [n, 3] float32."""
    L = lib()
    L.orc_deskew_scan.restype = None
    r = np.ascontiguousarray(ranges, np.float32)
    out = np.zeros((len(r), 3), np.float32)
    fp = C.POINTER(C.c_float)
    L.orc_deskew_scan(len(r), r.ctypes.data_as(fp), C.c_double(angle_min), C.c_double(angle_increment), C.byref(info),
                      _d(f64(imu_time)), _d(f64(rot_x)), _d(f64(rot_y)), _d(f64(rot_z)), out.ctypes.data_as(fp))
    return out
