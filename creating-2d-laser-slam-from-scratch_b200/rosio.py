"""ctypes harness over the C ABI — ROS-shaped input adapters (b2s_ros_*)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .matcher import check, lib


class LaserScanMsg(C.Structure):
    """b2s_laser_scan_msg: the sensor_msgs/LaserScan fields the lesson nodes read."""
    _fields_ = [("angle_min", C.c_float), ("angle_max", C.c_float), ("angle_increment", C.c_float),
                ("range_min", C.c_float), ("range_max", C.c_float), ("n_ranges", C.c_int32),
                ("ranges", C.POINTER(C.c_float))]


def make_msg(angle_min, angle_max, angle_increment, range_min, range_max, ranges):
    r = np.ascontiguousarray(ranges, np.float32)
    m = LaserScanMsg(angle_min, angle_max, angle_increment, range_min, range_max, len(r), r.ctypes.data_as(C.POINTER(C.c_float)))
    m._keep = r
    return m


def karto_laser(msg, laser_pose_in_base=(0.0, 0.0, 0.0), use_scan_range=12.0) -> abi.Laser:
    out = abi.Laser()
    pose = (C.c_double * 3)(*laser_pose_in_base)
    check(lib().b2s_ros_karto_laser(C.byref(msg), pose, C.c_double(use_scan_range), C.byref(out)))
    return out


def karto_readings(msg, inverted=False):
    out = np.zeros(msg.n_ranges)
    check(lib().b2s_ros_karto_readings(C.byref(msg), int(inverted), out.ctypes.data_as(C.POINTER(C.c_double))))
    return out


def hector_points(points_xyz, laser_in_base=(0, 0, 0, 0), scale_to_map=20.0, min_dist=0.2, max_dist=30.0,
                  use_max_scan_range=20.0, z_min=-1.0, z_max=1.0):
    p = np.ascontiguousarray(points_xyz, np.float32).reshape(-1, 3)
    out, origo, n = np.zeros((len(p), 2), np.float32), np.zeros(2, np.float32), C.c_int32(0)
    lib().b2s_ros_hector_points.argtypes = [C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float), C.c_float, C.c_float, C.c_float,
                                            C.c_double, C.c_float, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                            C.POINTER(C.c_int32)]
    lb = np.ascontiguousarray(laser_in_base, np.float32)
    fp = C.POINTER(C.c_float)
    check(lib().b2s_ros_hector_points(p.ctypes.data_as(fp), len(p), lb.ctypes.data_as(fp), scale_to_map, min_dist, max_dist,
                                      use_max_scan_range, z_min, z_max, out.ctypes.data_as(fp), origo.ctypes.data_as(fp), C.byref(n)))
    return out[:n.value].copy(), origo


class HectorScanFilter(C.Structure):
    """b2s_hector_scan_filter: HectorMappingRos::scanCallback's settings (node defaults)."""
    _fields_ = [("laser_in_base", C.c_float * 4), ("range_cutoff", C.c_double), ("use_max_scan_range", C.c_double),
                ("min_dist", C.c_float), ("max_dist", C.c_float), ("z_min", C.c_float), ("z_max", C.c_float)]


def hector_scan_filter(laser_in_base=(0, 0, 0, 0), range_cutoff=30.0, use_max_scan_range=20.0, min_dist=0.2,
                       max_dist=30.0, z_min=-1.0, z_max=1.0) -> HectorScanFilter:
    return HectorScanFilter((C.c_float * 4)(*laser_in_base), range_cutoff, use_max_scan_range, min_dist, max_dist, z_min, z_max)


def hector_scans(geometry, ranges, filt=None, scale_to_map=20.0):
    """b2s_ros_hector_scans: [n_scans, n_ranges] float32 ranges of one laser (geometry: a LaserScanMsg, its ranges
    ignored) -> (packed points [sum n][2], per-scan counts [n_scans], origo [2]), the DataContainers the node builds."""
    r = np.ascontiguousarray(ranges, np.float32).reshape(-1, geometry.n_ranges) if geometry.n_ranges else \
        np.zeros((len(ranges), 0), np.float32)
    n_scans = len(r)
    filt = filt if filt is not None else hector_scan_filter()
    out = np.zeros((max(r.size, 1), 2), np.float32)
    cnt, origo = np.zeros(n_scans, np.int32), np.zeros(2, np.float32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    L = lib()
    L.b2s_ros_hector_scans.argtypes = [C.POINTER(LaserScanMsg), C.POINTER(HectorScanFilter), C.c_float, C.c_int, fp, fp, ip, fp]
    check(L.b2s_ros_hector_scans(C.byref(geometry), C.byref(filt), scale_to_map, n_scans, r.ctypes.data_as(fp),
                                 out.ctypes.data_as(fp), cnt.ctypes.data_as(ip), origo.ctypes.data_as(fp)))
    return out[:int(cnt.sum())].copy(), cnt, origo
