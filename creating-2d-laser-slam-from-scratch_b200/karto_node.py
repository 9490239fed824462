"""ctypes harness over the C ABI — lesson6's SlamKarto node over whole recordings (b2s_karto_node_*)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .matcher import check, lib
from .mapper import Mapper, MapperParams, ScanSolver, _bind as _bind_mapper
from .rosio import LaserScanMsg

THROTTLED, NO_ODOM, NOT_MOVED, PROCESSED = 0, 1, 2, 3


class KartoNodeParams(C.Structure):
    """b2s_karto_node_params: the node's own parameters and the Mapper's values as it stores them."""
    _fields_ = [("throttle_scans", C.c_int32), ("reserved", C.c_int32), ("map_update_interval", C.c_double),
                ("resolution", C.c_double), ("use_scan_range", C.c_double), ("mapper", MapperParams)]


MAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.POINTER(abi.OccGridInfo), C.POINTER(C.c_int8))
BATCH_MAP_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(abi.OccGridInfo), C.POINTER(C.c_int8))

# SlamKarto::InitParams (karto_slam.cc:81-252): ROS parameter -> (where the Mapper stores it, type, squared by setParam*).
# minimum_time_interval is absent: the node never reads it.
_MAPPER_PARAMS = {
    "use_scan_matching": ("use_scan_matching", bool, False),
    "use_scan_barycenter": ("use_scan_barycenter", bool, False),
    "minimum_travel_distance": ("minimum_travel_distance", float, False),
    "minimum_travel_heading": ("minimum_travel_heading", float, False),
    "scan_buffer_size": ("scan_buffer_size", int, False),
    "scan_buffer_maximum_scan_distance": ("scan_buffer_maximum_scan_distance", float, False),
    "link_match_minimum_response_fine": ("link_match_minimum_response_fine", float, False),
    "link_scan_maximum_distance": ("link_scan_maximum_distance", float, False),
    "loop_search_maximum_distance": ("loop_search_maximum_distance", float, False),
    "do_loop_closing": ("do_loop_closing", bool, False),
    "loop_match_minimum_chain_size": ("loop_match_minimum_chain_size", int, False),
    "loop_match_maximum_variance_coarse": ("loop_match_maximum_variance_coarse", float, True),
    "loop_match_minimum_response_coarse": ("loop_match_minimum_response_coarse", float, False),
    "loop_match_minimum_response_fine": ("loop_match_minimum_response_fine", float, False),
    "correlation_search_space_dimension": ("sequential.search_size", float, False),
    "correlation_search_space_resolution": ("sequential.resolution", float, False),
    "correlation_search_space_smear_deviation": ("sequential.smear_deviation", float, False),
    "loop_search_space_dimension": ("loop.search_size", float, False),
    "loop_search_space_resolution": ("loop.resolution", float, False),
    "loop_search_space_smear_deviation": ("loop.smear_deviation", float, False),
    "distance_variance_penalty": ("*.distance_variance_penalty", float, True),
    "angle_variance_penalty": ("*.angle_variance_penalty", float, True),
    "fine_search_angle_offset": ("*.fine_search_angle_offset", float, False),
    "coarse_search_angle_offset": ("*.coarse_search_angle_offset", float, False),
    "coarse_angle_resolution": ("*.coarse_angle_resolution", float, False),
    "minimum_angle_penalty": ("*.minimum_angle_penalty", float, False),
    "minimum_distance_penalty": ("*.minimum_distance_penalty", float, False),
    "use_response_expansion": ("*.use_response_expansion", bool, False),
}


def node_params(ros: dict | None = None):
    """SlamKarto::InitParams over a ROS parameter dict (e.g. the parsed config/mapper_params.yaml): absent parameters keep
    the node's defaults and Mapper::InitializeParameters'; present ones go through the setParam* semantics, squaring
    included.  -> (KartoNodeParams, use_back_end)."""
    ros = dict(ros or {})
    p = KartoNodeParams()
    _bind_mapper().b2s_mapper_default_params(C.byref(p.mapper), float(ros.get("use_scan_range", 12.0)))
    p.throttle_scans = int(ros.get("throttle_scans", 1))
    p.map_update_interval = float(ros.get("map_update_interval", 5.0))
    p.resolution = float(ros.get("resolution", 0.05))
    p.use_scan_range = float(ros.get("use_scan_range", 12.0))
    for key, (field, kind, squared) in _MAPPER_PARAMS.items():
        if key not in ros:
            continue
        v = kind(ros[key])
        if squared:
            v = v * v  # math::Square
        if kind is bool:
            v = int(v)
        if field.startswith("*."):
            setattr(p.mapper.sequential, field[2:], v)
            setattr(p.mapper.loop, field[2:], v)
        elif "." in field:
            part, name = field.split(".")
            setattr(getattr(p.mapper, part), name, v)
        else:
            setattr(p.mapper, field, v)
    return p, bool(ros.get("use_back_end", False))


_bound = False


def _bind():
    global _bound
    L = lib()
    _bind_mapper()
    if _bound:
        return L
    vp, dp = C.c_void_p, C.POINTER(C.c_double)
    L.b2s_karto_node_create.argtypes = [C.POINTER(KartoNodeParams), C.POINTER(LaserScanMsg), dp, C.POINTER(ScanSolver),
                                        C.c_int, C.POINTER(vp)]
    L.b2s_karto_node_destroy.argtypes = [vp]
    L.b2s_karto_node_destroy.restype = None
    L.b2s_karto_node_mapper.argtypes = [vp]
    L.b2s_karto_node_mapper.restype = vp
    L.b2s_karto_node_process.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_uint32), dp,
                                         C.POINTER(C.c_int32), dp, dp, C.POINTER(C.c_int32), MAP_FN, vp]
    L.b2s_karto_node_create_batch.argtypes = [C.c_int, C.POINTER(KartoNodeParams), C.POINTER(LaserScanMsg), dp,
                                              C.POINTER(ScanSolver), C.c_int, C.POINTER(vp)]
    L.b2s_karto_node_mapper_of.argtypes = [vp, C.c_int]
    L.b2s_karto_node_mapper_of.restype = vp
    L.b2s_karto_node_process_batch.argtypes = [vp, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_uint32),
                                               dp, C.POINTER(C.c_int32), dp, dp, C.POINTER(C.c_int32), BATCH_MAP_FN, vp]
    L.b2s_karto_node_last_timing.argtypes = [vp, dp]
    _bound = True
    return L


class _InnerMapper(Mapper):
    """The node's own Mapper (b2s_karto_node_mapper): the graph getters of mapper.Mapper, owned by the node."""

    def __init__(self, L, h, n):
        self.L, self.h, self.n, self._keep = L, C.c_void_p(h), n, []

    def close(self):
        self.h = C.c_void_p()


def _map_of(info_p, payload_p):
    i = info_p.contents
    info = dict(width=i.width, height=i.height, offset=np.array(i.offset[:]), resolution=i.resolution,
                width_step=i.width_step, data_size=i.data_size, cell_visits=int(i.cell_visits))
    data = np.ctypeslib.as_array(payload_p, shape=(i.height * i.width,)).reshape(i.height, i.width).copy()
    return info, data


class KartoNode:
    """Stand-in for one SlamKarto node: process(ranges, stamps, odom) per part of a recording."""

    def __init__(self, params: KartoNodeParams, geometry: LaserScanMsg, laser_mount, solver: ScanSolver | None = None,
                 device: int = 0):
        self.L = _bind()
        self.h = C.c_void_p()
        self.n_ranges = geometry.n_ranges
        mount = np.ascontiguousarray(laser_mount, np.float64)
        assert mount.shape == (7,)
        self._solver = solver  # the vtable's owner must outlive the node
        check(self.L.b2s_karto_node_create(C.byref(params), C.byref(geometry), mount.ctypes.data_as(C.POINTER(C.c_double)),
                                           C.byref(solver) if solver is not None else None, device, C.byref(self.h)))
        self.mapper = _InnerMapper(self.L, self.L.b2s_karto_node_mapper(self.h), self._n_readings(params, geometry))

    @staticmethod
    def _n_readings(params, geometry):
        return int(abi.karto_round((float(np.float32(geometry.angle_max)) - float(np.float32(geometry.angle_min))) /
                                   float(np.float32(geometry.angle_increment))))

    def process(self, ranges, stamps, odom, on_map=None):
        """ranges [S][n] float32, stamps [S][2] (sec, nsec), odom [S][7] (translation xyz + quaternion xyzw, NaN = lookup
        failed).  on_map(scan_index, info, payload) is called for each published map (payload is a copy).
        -> dict(state, pose, map_to_odom, map_published, maps=[(scan_index, info dict, payload)])."""
        r = np.ascontiguousarray(ranges, np.float32).reshape(-1, self.n_ranges)
        s = np.ascontiguousarray(stamps, np.uint32).reshape(len(r), 2)
        o = np.ascontiguousarray(odom, np.float64).reshape(len(r), 7)
        S = len(r)
        state, pub = np.zeros(S, np.int32), np.zeros(S, np.int32)
        pose, m2o = np.zeros((S, 3)), np.zeros((S, 7))
        maps = []

        def cb(user, scan_index, info_p, payload_p):
            info, data = _map_of(info_p, payload_p)
            maps.append((int(scan_index), info, data))
            if on_map is not None:
                on_map(int(scan_index), info, data)

        fn = MAP_FN(cb)
        i32 = C.POINTER(C.c_int32)
        check(self.L.b2s_karto_node_process(self.h, S, r.ctypes.data_as(C.POINTER(C.c_float)),
                                            s.ctypes.data_as(C.POINTER(C.c_uint32)), o.ctypes.data_as(C.POINTER(C.c_double)),
                                            state.ctypes.data_as(i32), pose.ctypes.data_as(C.POINTER(C.c_double)),
                                            m2o.ctypes.data_as(C.POINTER(C.c_double)), pub.ctypes.data_as(i32), fn, None))
        return dict(state=state, pose=pose, map_to_odom=m2o, map_published=pub, maps=maps)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.mapper.close()
            self.L.b2s_karto_node_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KartoNodeBatch:
    """B SlamKarto nodes in one handle, one per recording or per setting (b2s_karto_node_create_batch): their matches
    share launches and their maps are built together.  Every node must derive the same laser (offset, range threshold,
    upside-down flag) and the same matcher parameters; throttle, map interval, resolution, the Mapper's host-only
    parameters and the back end may differ.  solvers: None, or one ScanSolver (or None) per node, each its own."""

    def __init__(self, params_list, geometry: LaserScanMsg, mounts, solvers=None, device: int = 0):
        self.L = _bind()
        self.h = C.c_void_p()
        self.n_ranges = geometry.n_ranges
        self.batch = len(params_list)
        params = (KartoNodeParams * self.batch)(*params_list)
        m = np.ascontiguousarray(mounts, np.float64)
        assert m.shape == (self.batch, 7)
        slots = None
        if solvers is not None:
            assert len(solvers) == self.batch
            slots = (ScanSolver * self.batch)(*[s if s is not None else ScanSolver() for s in solvers])
        self._solvers = (solvers, slots)  # the vtables' owners must outlive the handle
        check(self.L.b2s_karto_node_create_batch(self.batch, params, C.byref(geometry),
                                                 m.ctypes.data_as(C.POINTER(C.c_double)), slots, device,
                                                 C.byref(self.h)))
        n = KartoNode._n_readings(params_list[0], geometry)
        self._mappers = [_InnerMapper(self.L, self.L.b2s_karto_node_mapper_of(self.h, b), n) for b in range(self.batch)]

    def mapper(self, b):
        """node b's Mapper (graph getters of mapper.Mapper)"""
        return self._mappers[b]

    def process(self, ranges_list, stamps_list, odom_list, on_map=None):
        """ranges_list[b] [S_b][n] float32, stamps_list[b] [S_b][2], odom_list[b] [S_b][7] -> one dict per node, shaped
        as KartoNode.process's.  on_map(node, scan_index, info, payload) is called for each published map in the call's
        order."""
        counts = np.array([len(s) for s in stamps_list], np.int32)
        assert len(counts) == self.batch and len(ranges_list) == self.batch and len(odom_list) == self.batch
        S = int(counts.sum())
        r = np.zeros((S, self.n_ranges), np.float32)
        s = np.zeros((S, 2), np.uint32)
        o = np.zeros((S, 7), np.float64)
        at = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        for b in range(self.batch):
            if counts[b]:
                r[at[b]:at[b + 1]] = np.asarray(ranges_list[b], np.float32).reshape(counts[b], self.n_ranges)
                s[at[b]:at[b + 1]] = np.asarray(stamps_list[b], np.uint32).reshape(counts[b], 2)
                o[at[b]:at[b + 1]] = np.asarray(odom_list[b], np.float64).reshape(counts[b], 7)
        state, pub = np.zeros(S, np.int32), np.zeros(S, np.int32)
        pose, m2o = np.zeros((S, 3)), np.zeros((S, 7))
        maps = [[] for _ in range(self.batch)]

        def cb(user, node, scan_index, info_p, payload_p):
            info, data = _map_of(info_p, payload_p)
            maps[node].append((int(scan_index), info, data))
            if on_map is not None:
                on_map(int(node), int(scan_index), info, data)

        fn = BATCH_MAP_FN(cb)
        i32, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
        check(self.L.b2s_karto_node_process_batch(self.h, counts.ctypes.data_as(i32), r.ctypes.data_as(C.POINTER(C.c_float)),
                                                  s.ctypes.data_as(C.POINTER(C.c_uint32)), o.ctypes.data_as(dp),
                                                  state.ctypes.data_as(i32), pose.ctypes.data_as(dp),
                                                  m2o.ctypes.data_as(dp), pub.ctypes.data_as(i32), fn, None))
        return [dict(state=state[at[b]:at[b + 1]], pose=pose[at[b]:at[b + 1]], map_to_odom=m2o[at[b]:at[b + 1]],
                     map_published=pub[at[b]:at[b + 1]], maps=maps[b]) for b in range(self.batch)]

    def last_timing(self):
        """where the last process call went (b2s_karto_node_last_timing)"""
        out = np.zeros(8)
        check(self.L.b2s_karto_node_last_timing(self.h, out.ctypes.data_as(C.POINTER(C.c_double))))
        keys = ("rounds", "match_launches", "matches", "maps", "match_s", "map_s", "map_bytes_d2h", "call_s")
        return dict(zip(keys, out.tolist()))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            for m in self._mappers:
                m.close()
            self.L.b2s_karto_node_destroy(self.h)
            self.h = C.c_void_p()

    __del__ = KartoNode.__del__
