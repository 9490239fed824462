"""ctypes harness over the C ABI — lesson5 motion de-skew (LidarUndistortion, lidar_undistortion.cc): the batched
CorrectLaserScan on the device plus the per-scan host preparation (IMU angle integration, odometry increment)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .matcher import check, lib, f64, _d


class DeskewScan(C.Structure):
    """b2s_deskew_scan (include/b200slam.h)."""
    _fields_ = [("time_start", C.c_double), ("time_increment", C.c_double), ("range_min", C.c_float), ("range_max", C.c_float),
                ("use_imu", C.c_int32), ("use_odom", C.c_int32), ("imu_last", C.c_int32), ("reserved", C.c_int32),
                ("odom_start_time", C.c_double), ("odom_end_time", C.c_double), ("odom_incre", C.c_float * 3),
                ("reserved2", C.c_float)]


class ImuMsg(C.Structure):
    """b2s_imu_msg: header.stamp and angular_velocity of a sensor_msgs/Imu."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("angular_velocity", C.c_double * 3)]


class OdomMsg(C.Structure):
    """b2s_odom_msg: header.stamp, pose.pose.position and pose.pose.orientation (x, y, z, w) of a nav_msgs/Odometry."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("position", C.c_double * 3), ("orientation", C.c_double * 4)]


class NodeScan(C.Structure):
    """b2s_deskew_node_scan: one LaserScan's per-scan fields and the messages delivered before its callback."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("time_increment", C.c_float), ("range_min", C.c_float),
                ("range_max", C.c_float), ("imu_arrived", C.c_int32), ("odom_arrived", C.c_int32),
                ("reserved", C.c_int32)]


# numpy record layouts of the structs, for whole logs
IMU_DTYPE, ODOM_DTYPE, SCAN_DTYPE, STATE_DTYPE = (np.dtype(s) for s in (ImuMsg, OdomMsg, NodeScan, DeskewScan))
# B2S_DESKEW_* (include/b200slam.h)
PUBLISHED, HELD, WAIT_IMU, IMU_EMPTY, WAIT_ODOM, ODOM_EMPTY, UNDEFINED = range(7)


def imu_log(stamps, angular_velocity):
    """stamps [N, 2] (sec, nsec), angular_velocity [N, 3] -> IMU_DTYPE [N]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), IMU_DTYPE)
    a["sec"], a["nsec"], a["angular_velocity"] = st[:, 0], st[:, 1], np.asarray(angular_velocity, np.float64).reshape(-1, 3)
    return a


def odom_log(stamps, position, orientation):
    """stamps [N, 2], position [N, 3], orientation [N, 4] (x, y, z, w) -> ODOM_DTYPE [N]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), ODOM_DTYPE)
    a["sec"], a["nsec"] = st[:, 0], st[:, 1]
    a["position"], a["orientation"] = np.asarray(position).reshape(-1, 3), np.asarray(orientation).reshape(-1, 4)
    return a


def node_scans(stamps, time_increment, range_min, range_max, imu_arrived, odom_arrived):
    """per-scan stamps [S, 2] (sec, nsec), float fields (scalars or [S]) and arrival counts [S] -> SCAN_DTYPE [S]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), SCAN_DTYPE)
    a["sec"], a["nsec"] = st[:, 0], st[:, 1]
    a["time_increment"], a["range_min"], a["range_max"] = time_increment, range_min, range_max
    a["imu_arrived"], a["odom_arrived"] = imu_arrived, odom_arrived
    return a


_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
        L.b2s_deskew_integrate_imu.argtypes = [C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, dp, dp, dp, dp]
        L.b2s_deskew_integrate_imu.restype = C.c_int32
        L.b2s_deskew_odom_increment.argtypes = [dp, dp, fp]
        L.b2s_deskew_odom_increment.restype = None
        L.b2s_lidar_undistort.argtypes = [C.c_int, C.c_int, fp, C.c_double, C.c_double, C.POINTER(DeskewScan), dp, dp, dp, dp,
                                          C.c_int, fp, C.c_int, C.c_void_p]
        vp = C.c_void_p
        L.b2s_lidar_undistortion_node.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, vp, vp, C.c_int,
                                                  vp, C.c_int, vp, vp, vp, vp, C.c_int, vp]
        _bound = True
    return L


def integrate_imu(stamps, angular_velocity, scan_start, scan_end, capacity=2000, fn=None):
    """PruneImuDeque's integration -> (imu_last, imu_time, rot_x, rot_y, rot_z)."""
    fn = fn or _bind().b2s_deskew_integrate_imu
    st, av = f64(stamps), f64(angular_velocity).reshape(-1, 3)
    t, x, y, z = (np.zeros(capacity) for _ in range(4))
    last = fn(len(st), _d(st), _d(av), float(scan_start), float(scan_end), capacity, _d(t), _d(x), _d(y), _d(z))
    return int(last), t, x, y, z


def odom_increment(start_pose, end_pose, fn=None):
    fn = fn or _bind().b2s_deskew_odom_increment
    out = np.zeros(3, np.float32)
    fn(_d(f64(start_pose)), _d(f64(end_pose)), out.ctypes.data_as(C.POINTER(C.c_float)))
    return out


def undistort(ranges, angle_min, angle_increment, scans, imu_time, rot_x, rot_y, rot_z, device=0, stream=None):
    """ranges [B, n] float32, scans: list of DeskewScan, IMU tables [B, stride] -> corrected cloud [B, n, 3] float32."""
    L = _bind()
    r = np.ascontiguousarray(ranges, np.float32)
    B, n = r.shape
    arr = (DeskewScan * B)(*scans)
    t, x, y, z = (np.ascontiguousarray(a, np.float64).reshape(B, -1) for a in (imu_time, rot_x, rot_y, rot_z))
    out = np.zeros((B, n, 3), np.float32)
    fp = C.POINTER(C.c_float)
    check(L.b2s_lidar_undistort(B, n, r.ctypes.data_as(fp), float(angle_min), float(angle_increment), arr, _d(t), _d(x), _d(y),
                                _d(z), t.shape[1], out.ctypes.data_as(fp), device, C.c_void_p(stream) if stream else None))
    return out


def undistort_recording(use_imu, use_odom, angle_min, angle_increment, scans, ranges, imu=(), odom=(), device=0,
                        stream=None, out=None):
    """The whole node over one recording (b2s_lidar_undistortion_node).  scans: SCAN_DTYPE [S] (node_scans), ranges
    [S, n] float32, imu / odom: IMU_DTYPE / ODOM_DTYPE logs in delivery order.  out: an optional float32 [S, n, 3]
    array for the clouds (page-locked memory speeds the copy).  -> (status [S] int32, state [S] STATE_DTYPE,
    xyz [S, n, 3] float32): rows are indexed by the corrected scan."""
    L = _bind()
    r = np.ascontiguousarray(ranges, np.float32)
    S, n = r.shape
    sc = np.ascontiguousarray(scans, SCAN_DTYPE)
    im, od = np.ascontiguousarray(imu, IMU_DTYPE), np.ascontiguousarray(odom, ODOM_DTYPE)
    assert len(sc) == S
    status, state = np.zeros(S, np.int32), np.zeros(S, STATE_DTYPE)
    xyz = np.zeros((S, n, 3), np.float32) if out is None else out
    assert xyz.dtype == np.float32 and xyz.shape == (S, n, 3) and xyz.flags.c_contiguous
    check(L.b2s_lidar_undistortion_node(int(use_imu), int(use_odom), float(angle_min), float(angle_increment), n, S,
                                        sc.ctypes.data, r.ctypes.data, len(im), im.ctypes.data, len(od), od.ctypes.data,
                                        status.ctypes.data,
                                        state.ctypes.data, xyz.ctypes.data, device, stream))
    return status, state, xyz
