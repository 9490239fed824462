"""TEST INFRASTRUCTURE — ctypes binding of oracle/liblesson4_nodes_oracle.so: the plain-C CPU restatement of lesson4's two
make-map nodes (lesson4_nodes_oracle.c) together with the GMapping and Hector map restatements it calls
(gmapping_oracle.c, hector_oracle.c), a library of its own built by oracle/recipes.py.  Only tests/, __graft_entry__ and
tools/ may import this module; the product never does.
"""
from __future__ import annotations

import ctypes as C
import importlib

import numpy as np

from oracle import recipes

node_maps = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.node_maps")

SENTINEL = 0x55  # an overrun byte the node does not write
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.build("liblesson4_nodes_oracle.so"))
        vp = C.c_void_p
        L.orc_gmapping_node_dims.argtypes = [vp, vp]
        L.orc_gmapping_node_maps.argtypes = [vp, vp, C.c_int, vp, vp, vp, C.c_int, vp]
        L.orc_hector_mapping_node_dims.argtypes = [vp, vp]
        L.orc_hector_mapping_node_maps.argtypes = [vp, vp, C.c_int, vp, vp]
        _lib = L
    return _lib


def _ranges(ranges):
    r = np.ascontiguousarray(ranges, np.float32)
    assert r.ndim == 2
    return r


def gmapping_dims(params) -> tuple:
    d = np.zeros(2, np.int32)
    if lib().orc_gmapping_node_dims(C.addressof(params), d.ctypes.data):
        raise ValueError("bounds the node cannot size")
    return int(d[0]), int(d[1])


def gmapping(fields, params, ranges, overrun_cap=0):
    """The node's published maps for every scan.  fields = (angle_min, angle_increment, range_min, range_max) float32,
    params a node_maps.GMappingNodeParams, ranges [S][n] float32.  -> (maps [S][height][width] int8, first refused
    scan or S, overrun [S][overrun_cap] int8, n_overrun [S])."""
    r = _ranges(ranges)
    w, h = gmapping_dims(params)
    geom = node_maps.geometry(*fields, r.shape[1])
    maps = np.zeros((len(r), h, w), np.int8)
    ov = np.zeros((len(r), max(overrun_cap, 0)), np.int8)
    nov = np.zeros(len(r), np.int32)
    first = lib().orc_gmapping_node_maps(C.addressof(geom), C.addressof(params), len(r), r.ctypes.data, maps.ctypes.data,
                                         ov.ctypes.data if overrun_cap > 0 else None, overrun_cap, nov.ctypes.data)
    return maps, first, ov, nov


def hector_dims(params) -> tuple:
    d = np.zeros(2, np.int32)
    if lib().orc_hector_mapping_node_dims(C.addressof(params), d.ctypes.data):
        raise ValueError("bounds the node cannot size")
    return int(d[0]), int(d[1])


def hector(fields, params, ranges) -> np.ndarray:
    """The node's published maps [S][height][width] int8 for every scan (arguments as for gmapping)."""
    r = _ranges(ranges)
    w, h = hector_dims(params)
    geom = node_maps.geometry(*fields, r.shape[1])
    maps = np.zeros((len(r), h, w), np.int8)
    assert lib().orc_hector_mapping_node_maps(C.addressof(geom), C.addressof(params), len(r), r.ctypes.data,
                                              maps.ctypes.data) == 0
    return maps
