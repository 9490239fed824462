"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson5_ref.so: the UNMODIFIED lesson5 node,
reference/lesson5/src/lidar_undistortion.cc, compiled where it lies against the ROS, tf, PCL and Eigen stand-ins under
oracle/shim/ by oracle/ref_lesson5.cpp, built by oracle/recipes.py from a checkout of the original project; where it
is absent the tests replay its recorded answers (tests/reference_record.py).  Only tests/ and __graft_entry__ may import
this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/liblesson5_ref.so"
QUEUE_LENGTH = 2000  # the node's imu table length (lidar_undistortion.cc:20)
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        u32, dp, fp = C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_float)
        L.ref_deskew_new.argtypes = [C.c_int, C.c_int]
        L.ref_deskew_new.restype = None
        L.ref_deskew_imu.argtypes = [u32, u32, C.c_double, C.c_double, C.c_double]
        L.ref_deskew_imu.restype = None
        L.ref_deskew_odom.argtypes = [u32, u32, dp, dp]
        L.ref_deskew_odom.restype = None
        L.ref_deskew_scan.argtypes = [u32, u32, fp, C.c_int, fp]
        L.ref_deskew_scan.restype = C.c_int
        L.ref_deskew_published.argtypes = [C.POINTER(u32), dp, dp, fp, C.c_int, fp, C.c_int, dp, dp, dp, dp]
        L.ref_deskew_published.restype = C.c_int
        _lib = L
    return _lib


def run(events, use_imu: bool, use_odom: bool) -> list:
    """Feed one message stream to a fresh node and collect every cloud it publishes.

    events: ("imu", sec, nsec, (wx, wy, wz)) | ("odom", sec, nsec, (x, y, z), (qx, qy, qz, qw))
            | ("scan", sec, nsec, (angle_min, angle_increment, time_increment, range_min, range_max), ranges[n])
    -> one dict per published cloud: stamp [sec, nsec], times [scan start, scan end, odometry start, odometry end],
       poses [2, 6] (x, y, z, roll, pitch, yaw of the odometry messages the node chose), incre [3] (float32),
       xyz [n, 3] (float32), imu_last, imu [4, imu_last + 1] (time, rot x, y, z of the node's table)."""
    L = lib()
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    L.ref_deskew_new(int(use_imu), int(use_odom))
    out = []
    for e in events:
        if e[0] == "imu":
            L.ref_deskew_imu(e[1], e[2], *map(float, e[3]))
        elif e[0] == "odom":
            pos, quat = np.ascontiguousarray(e[3], np.float64), np.ascontiguousarray(e[4], np.float64)
            L.ref_deskew_odom(e[1], e[2], pos.ctypes.data_as(dp), quat.ctypes.data_as(dp))
        else:
            fields, r = np.ascontiguousarray(e[3], np.float32), np.ascontiguousarray(e[4], np.float32)
            if not L.ref_deskew_scan(e[1], e[2], fields.ctypes.data_as(fp), len(r), r.ctypes.data_as(fp)):
                continue
            stamp, times, poses, incre = np.zeros(2, np.uint32), np.zeros(4), np.zeros(12), np.zeros(3, np.float32)
            xyz = np.zeros((len(r), 3), np.float32)
            tab = np.zeros((4, QUEUE_LENGTH))
            last = L.ref_deskew_published(stamp.ctypes.data_as(C.POINTER(C.c_uint32)), times.ctypes.data_as(dp),
                                          poses.ctypes.data_as(dp), incre.ctypes.data_as(fp), len(r), xyz.ctypes.data_as(fp),
                                          QUEUE_LENGTH, *(tab[k].ctypes.data_as(dp) for k in range(4)))
            out.append(dict(stamp=stamp, times=times, poses=poses.reshape(2, 6), incre=incre, xyz=xyz, imu_last=int(last),
                            imu=np.ascontiguousarray(tab[:, :max(last, 0) + 1])))
    return out
