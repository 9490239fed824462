"""ctypes harness over the C ABI — lesson4's Hector SLAM node over whole recordings (b2s_hector_node_*)."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from .hector import _bind as _bind_hector
from .matcher import check, lib
from .rosio import LaserScanMsg


class HectorNodeParams(C.Structure):
    """b2s_hector_node_params: the values HectorMappingRos::InitParams stores, in the node's types."""
    _fields_ = [("map_resolution", C.c_double), ("map_size", C.c_int32), ("map_multi_res_levels", C.c_int32),
                ("map_start_x", C.c_double), ("map_start_y", C.c_double), ("update_factor_free", C.c_double),
                ("update_factor_occupied", C.c_double), ("map_update_distance_thresh", C.c_double),
                ("map_update_angle_thresh", C.c_double), ("use_max_scan_range", C.c_double),
                ("laser_min_dist", C.c_double), ("laser_max_dist", C.c_double), ("laser_z_min_value", C.c_float),
                ("laser_z_max_value", C.c_float), ("map_pub_period", C.c_double)]


class HectorNodeMapInfo(C.Structure):
    """b2s_hector_node_map_info: the MapMetaData setMapInfo fills."""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_float), ("width", C.c_int32),
                ("height", C.c_int32)]


MAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.POINTER(C.c_uint32), C.POINTER(HectorNodeMapInfo),
                     C.POINTER(C.c_int8), C.c_int32)
BATCH_MAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_uint32), C.POINTER(HectorNodeMapInfo),
                           C.POINTER(C.c_int8), C.c_int32)

# HectorMappingRos::InitParams (hector_slam.cc:119-162): ROS parameter -> (field, type, node default)
_PARAMS = {
    "map_resolution": ("map_resolution", float, 0.05),
    "map_size": ("map_size", int, 2048),
    "map_start_x": ("map_start_x", float, 0.5),
    "map_start_y": ("map_start_y", float, 0.5),
    "map_multi_res_levels": ("map_multi_res_levels", int, 3),
    "update_factor_free": ("update_factor_free", float, 0.4),
    "update_factor_occupied": ("update_factor_occupied", float, 0.9),
    "map_update_distance_thresh": ("map_update_distance_thresh", float, 0.4),
    "map_update_angle_thresh": ("map_update_angle_thresh", float, 0.9),
    "use_max_scan_range": ("use_max_scan_range", float, 20.0),
    "laser_min_dist": ("laser_min_dist", float, 0.2),
    "laser_max_dist": ("laser_max_dist", float, 30.0),
    "laser_z_min_value": ("laser_z_min_value", float, -1.0),
    "laser_z_max_value": ("laser_z_max_value", float, 1.0),
    "map_pub_period": ("map_pub_period", float, 2.0),
}

# lesson4/launch/hector_slam.launch's node parameters (the frame, topic and publish switches aside).  It writes
# map_multi_res_levels as "３" (U+FF13, a full-width digit); see node_params for what that becomes.
SHIPPED_LAUNCH = {"use_max_scan_range": "20", "laser_min_dist": "0.2", "laser_max_dist": "30", "map_pub_period": "2",
                  "map_resolution": "0.05", "map_multi_res_levels": "３", "map_update_distance_thresh": "0.4",
                  "map_update_angle_thresh": "0.9"}

# a laser mounted as the shipped launch does: static_transform_publisher 0 0 0.254 0 0 3.1415926, whose arguments are
# x y z yaw pitch roll, so the laser is upside down (roll pi).  Quaternion::setRPY(3.1415926, 0, 0) in double:
# x = sin(roll * 0.5), y = z = 0, w = cos(roll * 0.5)
SHIPPED_MOUNT = (0.0, 0.0, 0.254, math.sin(3.1415926 * 0.5), 0.0, 0.0, math.cos(3.1415926 * 0.5))


def node_params(ros: dict | None = None) -> HectorNodeParams:
    """HectorMappingRos::InitParams over a ROS parameter dict: absent keys keep the node's defaults; present ones are
    converted as roslaunch's automatic typing does, with Python's int() / float().  Python's int() reads the launch
    file's full-width "３" as 3, which is also the default, so map_multi_res_levels is 3 either way.  The laser
    distances stay in metres: the handle squares them in double as the node does."""
    ros = dict(ros or {})
    p = HectorNodeParams()
    for key, (field, kind, default) in _PARAMS.items():
        v = ros.get(key, default)
        setattr(p, field, kind(v))
    return p


_bound = False


def _bind():
    global _bound
    L = lib()
    _bind_hector()
    if _bound:
        return L
    vp, fp, dp, ip = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
    L.b2s_hector_node_create.argtypes = [C.POINTER(HectorNodeParams), C.POINTER(LaserScanMsg), dp, C.c_int, C.POINTER(vp)]
    L.b2s_hector_node_destroy.argtypes = [vp]
    L.b2s_hector_node_destroy.restype = None
    L.b2s_hector_node_processor.argtypes = [vp]
    L.b2s_hector_node_processor.restype = vp
    L.b2s_hector_node_process.argtypes = [vp, C.c_int, fp, C.POINTER(C.c_uint32), fp, dp, dp, ip, ip, MAP_FN, vp]
    L.b2s_hector_node_publish_map.argtypes = [vp, C.POINTER(C.c_uint32), MAP_FN, vp]
    L.b2s_hector_node_create_batch.argtypes = [C.c_int, C.POINTER(HectorNodeParams), C.POINTER(LaserScanMsg), dp, C.c_int,
                                               C.POINTER(vp)]
    L.b2s_hector_node_process_batch.argtypes = [vp, ip, fp, C.POINTER(C.c_uint32), fp, dp, dp, ip, ip, BATCH_MAP_FN, vp]
    L.b2s_hector_node_publish_map_of.argtypes = [vp, C.c_int, C.POINTER(C.c_uint32), BATCH_MAP_FN, vp]
    L.b2s_hector_node_create_fleet.argtypes = [C.c_int, C.POINTER(HectorNodeParams), C.POINTER(LaserScanMsg), dp, C.c_int,
                                               C.POINTER(vp)]
    _bound = True
    return L


def _map_dict(scan_index, stamp_p, info_p, payload_p, rebuilt):
    i = info_p.contents
    info = dict(origin_x=i.origin_x, origin_y=i.origin_y, resolution=i.resolution, width=i.width, height=i.height)
    data = np.ctypeslib.as_array(payload_p, shape=(i.height * i.width,)).reshape(i.height, i.width).copy()
    return dict(scan_index=int(scan_index), stamp=(int(stamp_p[0]), int(stamp_p[1])), info=info, payload=data,
                rebuilt=bool(rebuilt))


def _collector(maps, on_map):
    def cb(user, scan_index, stamp_p, info_p, payload_p, rebuilt):
        m = _map_dict(scan_index, stamp_p, info_p, payload_p, rebuilt)
        if on_map is not None:
            on_map(m)
        else:
            maps.append(m)
    return MAP_FN(cb)


def _batch_collector(maps, on_map):
    """maps: one list per node; on_map(node, dict) instead when given"""
    def cb(user, node, scan_index, stamp_p, info_p, payload_p, rebuilt):
        m = _map_dict(scan_index, stamp_p, info_p, payload_p, rebuilt)
        if on_map is not None:
            on_map(int(node), m)
        else:
            maps[node].append(m)
    return BATCH_MAP_FN(cb)


class HectorNode:
    """Stand-in for one HectorMappingRos: process(ranges, stamps) per part of a recording."""

    def __init__(self, params: HectorNodeParams, geometry: LaserScanMsg, laser_mount=(0, 0, 0, 0, 0, 0, 1), device=0):
        self.L = _bind()
        self.h = C.c_void_p()
        self.n_ranges = geometry.n_ranges
        mount = np.ascontiguousarray(laser_mount, np.float64)
        assert mount.shape == (7,)
        check(self.L.b2s_hector_node_create(C.byref(params), C.byref(geometry), mount.ctypes.data_as(C.POINTER(C.c_double)),
                                            device, C.byref(self.h)))
        self.processor = C.c_void_p(self.L.b2s_hector_node_processor(self.h))

    def process(self, ranges, stamps, on_map=None):
        """ranges [S][n] float32, stamps [S][2] (sec, nsec).  Maps go to on_map(dict) when given, else into the result.
        -> dict(pose [S,3] float32, pose_msg [S,7], cov [S,36], map_updated [S], n_points [S], maps [dict])."""
        r = np.ascontiguousarray(ranges, np.float32).reshape(-1, self.n_ranges) if self.n_ranges else \
            np.zeros((len(stamps), 0), np.float32)
        S = len(r)
        s = np.ascontiguousarray(stamps, np.uint32).reshape(S, 2)
        pose, msg, cov = np.zeros((S, 3), np.float32), np.zeros((S, 7)), np.zeros((S, 36))
        upd, kept = np.zeros(S, np.int32), np.zeros(S, np.int32)
        maps = []
        fn = _collector(maps, on_map)
        ip, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
        check(self.L.b2s_hector_node_process(self.h, S, r.ctypes.data_as(C.POINTER(C.c_float)),
                                             s.ctypes.data_as(C.POINTER(C.c_uint32)),
                                             pose.ctypes.data_as(C.POINTER(C.c_float)), msg.ctypes.data_as(dp),
                                             cov.ctypes.data_as(dp), upd.ctypes.data_as(ip), kept.ctypes.data_as(ip),
                                             fn, None))
        return dict(pose=pose, pose_msg=msg, cov=cov, map_updated=upd.astype(bool), n_points=kept, maps=maps)

    def publish_map(self, stamp):
        """publishMap now, stamped (sec, nsec) -> the map dict."""
        maps = []
        st = (C.c_uint32 * 2)(*stamp)
        check(self.L.b2s_hector_node_publish_map(self.h, st, _collector(maps, None), None))
        return maps[0]

    def level_ros(self, level=0):
        """The inner processor's level as a ROS payload (b2s_hector_slam_copy_level_ros)."""
        dims, cl = (C.c_int * 2)(), C.c_float(0)
        check(self.L.b2s_hector_slam_level_dims(self.processor, level, dims, C.byref(cl)))
        out = np.zeros((dims[1], dims[0]), np.int8)
        check(self.L.b2s_hector_slam_copy_level_ros(self.processor, level, out.ctypes.data_as(C.POINTER(C.c_int8))))
        return out

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.b2s_hector_node_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HectorNodeBatch:
    """B HectorMappingRos nodes in one handle, one per recording or per setting (b2s_hector_node_create_batch): the
    processor fields of every params set must be equal; mounts, range limits, z windows and periods may differ.
    HectorNodeBatch.fleet takes nodes with nothing in common."""

    def __init__(self, params_list, geometry: LaserScanMsg, mounts, device=0):
        self.L = _bind()
        self.h = C.c_void_p()
        self.batch = len(params_list)
        self.n_ranges = [geometry.n_ranges] * self.batch
        params = (HectorNodeParams * self.batch)(*params_list)
        m = np.ascontiguousarray(mounts, np.float64)
        assert m.shape == (self.batch, 7)
        check(self.L.b2s_hector_node_create_batch(self.batch, params, C.byref(geometry),
                                                  m.ctypes.data_as(C.POINTER(C.c_double)), device, C.byref(self.h)))
        self.processor = C.c_void_p(self.L.b2s_hector_node_processor(self.h))

    @classmethod
    def fleet(cls, params_list, geometries, mounts, device=0):
        """Nodes of different robots in one handle (b2s_hector_node_create_fleet): per node its own params (map size,
        resolution, levels, ... included), its own LaserScanMsg geometry and its own mount."""
        self = cls.__new__(cls)
        self.L = _bind()
        self.h = C.c_void_p()
        self.batch = len(params_list)
        assert len(geometries) == self.batch
        self.n_ranges = [g.n_ranges for g in geometries]
        params = (HectorNodeParams * self.batch)(*params_list)
        geoms = (LaserScanMsg * self.batch)(*geometries)
        m = np.ascontiguousarray(mounts, np.float64)
        assert m.shape == (self.batch, 7)
        check(self.L.b2s_hector_node_create_fleet(self.batch, params, geoms, m.ctypes.data_as(C.POINTER(C.c_double)),
                                                  device, C.byref(self.h)))
        self.processor = C.c_void_p(self.L.b2s_hector_node_processor(self.h))
        return self

    def process(self, ranges_list, stamps_list, on_map=None):
        """ranges_list[b] [S_b][n_b] float32 (n_b = node b's n_ranges), stamps_list[b] [S_b][2] -> one dict per node,
        shaped as HectorNode.process's.  Maps go to on_map(node, dict) in the call's order when given."""
        counts = np.array([len(s) for s in stamps_list], np.int32)
        assert len(counts) == self.batch and len(ranges_list) == self.batch
        S = int(counts.sum())
        r = np.concatenate([np.ascontiguousarray(ranges_list[b], np.float32).reshape(-1) if counts[b] else
                            np.zeros(0, np.float32) for b in range(self.batch)] + [np.zeros(0, np.float32)])
        assert len(r) == int((counts * np.array(self.n_ranges, np.int64)).sum())
        s = np.zeros((S, 2), np.uint32)
        at = np.concatenate([[0], np.cumsum(counts)])
        for b in range(self.batch):
            if counts[b]:
                s[at[b]:at[b + 1]] = np.asarray(stamps_list[b], np.uint32).reshape(counts[b], 2)
        pose, msg, cov = np.zeros((S, 3), np.float32), np.zeros((S, 7)), np.zeros((S, 36))
        upd, kept = np.zeros(S, np.int32), np.zeros(S, np.int32)
        maps = [[] for _ in range(self.batch)]
        fn = _batch_collector(maps, on_map)
        ip, dp, fp = C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_float)
        check(self.L.b2s_hector_node_process_batch(self.h, counts.ctypes.data_as(ip), r.ctypes.data_as(fp),
                                                   s.ctypes.data_as(C.POINTER(C.c_uint32)), pose.ctypes.data_as(fp),
                                                   msg.ctypes.data_as(dp), cov.ctypes.data_as(dp),
                                                   upd.ctypes.data_as(ip), kept.ctypes.data_as(ip), fn, None))
        return [dict(pose=pose[at[b]:at[b + 1]], pose_msg=msg[at[b]:at[b + 1]], cov=cov[at[b]:at[b + 1]],
                     map_updated=upd[at[b]:at[b + 1]].astype(bool), n_points=kept[at[b]:at[b + 1]], maps=maps[b])
                for b in range(self.batch)]

    def publish_map(self, b, stamp):
        """node b's publishMap now, stamped (sec, nsec) -> the map dict"""
        maps = [[] for _ in range(self.batch)]
        st = (C.c_uint32 * 2)(*stamp)
        check(self.L.b2s_hector_node_publish_map_of(self.h, b, st, _batch_collector(maps, None), None))
        return maps[b][0]

    def level_ros(self, b, level=0):
        """Node b's processor level as a ROS payload (b2s_hector_slam_copy_level_ros_of)."""
        dims, cl = (C.c_int * 2)(), C.c_float(0)
        check(self.L.b2s_hector_slam_level_dims_of(self.processor, b, level, dims, C.byref(cl)))
        out = np.zeros((dims[1], dims[0]), np.int8)
        check(self.L.b2s_hector_slam_copy_level_ros_of(self.processor, b, level, out.ctypes.data_as(C.POINTER(C.c_int8))))
        return out

    close = HectorNode.close
    __del__ = HectorNode.__del__
