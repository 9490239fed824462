"""ctypes harness over the C ABI — lesson4's make-map nodes over whole recordings: the GMapping node
(b2s_gmapping_node_maps, gmapping.cc) and the Hector make-map node (b2s_hector_mapping_node_maps, hector_mapping.cc)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .matcher import check, lib
from .rosio import LaserScanMsg

MAX_RANGES = 16384  # B2S_NODE_MAPS_MAX_RANGES
# the nodes' InitParams defaults (gmapping.cc:44-62, hector_mapping.cc:44-55)
GMAPPING_DEFAULTS = dict(max_range=30 - 0.01, max_use_range=25.0, xmin=-40.0, ymin=-40.0, xmax=40.0, ymax=40.0,
                         delta=0.05, occ_thresh=0.25)
HECTOR_DEFAULTS = dict(xmin=-40.0, ymin=-40.0, xmax=40.0, ymax=40.0, delta=0.05)


class GMappingNodeParams(C.Structure):
    """b2s_gmapping_node_params"""
    _fields_ = [(k, C.c_double) for k in ("max_range", "max_use_range", "xmin", "ymin", "xmax", "ymax", "delta",
                                          "occ_thresh")]


class HectorMappingNodeParams(C.Structure):
    """b2s_hector_mapping_node_params"""
    _fields_ = [(k, C.c_double) for k in ("xmin", "ymin", "xmax", "ymax")] + [("delta", C.c_float),
                                                                              ("reserved", C.c_float)]


def gmapping_params(**kw) -> GMappingNodeParams:
    return GMappingNodeParams(**{**GMAPPING_DEFAULTS, **kw})


def hector_params(**kw) -> HectorMappingNodeParams:
    return HectorMappingNodeParams(**{**HECTOR_DEFAULTS, **kw})


def geometry(angle_min, angle_increment, range_min, range_max, n_ranges) -> LaserScanMsg:
    """The b2s_laser_scan_msg of one laser (float32 fields; its ranges pointer is not read)."""
    a, inc = np.float32(angle_min), np.float32(angle_increment)
    return LaserScanMsg(a, a + inc * np.float32(max(n_ranges - 1, 0)), inc, range_min, range_max, n_ranges, None)


_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        vp = C.c_void_p
        for f, P in ((L.b2s_gmapping_node_maps, GMappingNodeParams), (L.b2s_hector_mapping_node_maps,
                                                                     HectorMappingNodeParams)):
            f.argtypes = [C.POINTER(LaserScanMsg), C.POINTER(P), C.c_int, vp, C.POINTER(C.c_int32), vp, C.c_int, vp]
        _bound = True
    return L


def _maps(fn, params, fields, ranges, out, device, stream):
    r = np.ascontiguousarray(ranges, np.float32)
    if r.ndim != 2:
        raise ValueError("ranges must be [n_scans][n_ranges]")
    geom = geometry(*fields, r.shape[1])
    dims = (C.c_int32 * 2)()
    check(fn(C.byref(geom), C.byref(params), len(r), None, dims, None, device, None))
    shape = (len(r), dims[1], dims[0])
    if out is None:
        out = np.empty(shape, np.int8)
    elif out.shape != shape or out.dtype != np.int8 or not out.flags.c_contiguous:
        raise ValueError(f"out must be a C-contiguous int8 array of shape {shape}")
    check(fn(C.byref(geom), C.byref(params), len(r), r.ctypes.data, dims, out.ctypes.data, device,
             C.c_void_p(stream) if stream else None))
    return out


def gmapping_maps(ranges, fields, params=None, out=None, device=0, stream=None) -> np.ndarray:
    """GMapping::ScanCallback on every scan of ranges [n_scans][n_ranges] float32 from one laser, fields =
    (angle_min, angle_increment, range_min, range_max) -> the published maps [n_scans][height][width] int8 (written
    into `out` when given, e.g. page-locked memory)."""
    return _maps(_bind().b2s_gmapping_node_maps, params or gmapping_params(), fields, ranges, out, device, stream)


def hector_maps(ranges, fields, params=None, out=None, device=0, stream=None) -> np.ndarray:
    """HectorMapping::ScanCallback on every scan (arguments as for gmapping_maps)."""
    return _maps(_bind().b2s_hector_mapping_node_maps, params or hector_params(), fields, ranges, out, device, stream)
