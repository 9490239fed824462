"""lesson6's Karto SLAM node on the device (b2s_karto_node_*) against the restatement oracle/karto_node_port.py, which
tests/test_karto_node_reference.py pins to the unmodified node: states and published-map flags exactly, corrected
poses and map_to_odom to 1e-9 (the device's sin / cos may differ from glibc's in the last place), graph edges exactly,
and every published payload byte-identical to the restated occupancy grid fed the node's own poses at that moment and
to the restatement's map.  Also: chunked calls equal one call, one node equals the per-scan route through
b2s_mapper_process_sensor and b2s_occ_grid_create_from_scans, and refused calls write nothing."""
import ctypes as C
import functools
import importlib

import numpy as np
import pytest

import karto_node_cases as kc
from oracle import karto_node_port, port

pytestmark = pytest.mark.gpu
KN = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.karto_node")
OG = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.occgrid")
MP = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.mapper")


@functools.lru_cache(maxsize=None)
def ported(name):
    c = kc.CASES[name]
    prm, ube = KN.node_params(c.params)
    node = karto_node_port.PortKartoNode(prm, c.geometry(), c.mount, kc.pose_graph() if ube else None)
    out = node.process(c.ranges, c.stamps, c.odom)
    out["edges"] = node.mapper.edges()
    return out


def device_node(c):
    prm, ube = KN.node_params(c.params)
    return KN.KartoNode(prm, c.geometry(), c.mount, kc.pose_graph() if ube else None)


@pytest.mark.parametrize("name", list(kc.CASES))
def test_device_node_equals_port(name):
    c, want = kc.CASES[name], ported(name)
    node = device_node(c)
    own = []

    def on_map(i, info, payload):  # the restated grid from the node's own poses, read while the node waits
        g = port.occupancy_grid(laser_of(c), readings_of(c, node), node.mapper.poses(), KN.node_params(c.params)[0].resolution)
        own.append((g, payload))

    got = node.process(c.ranges, c.stamps, c.odom, on_map=on_map)
    assert np.array_equal(got["state"], want["state"]) and np.array_equal(got["map_published"], want["map_published"])
    assert np.abs(got["pose"] - want["pose"]).max(initial=0.0) <= 1e-9
    assert np.abs(got["map_to_odom"] - want["map_to_odom"]).max(initial=0.0) <= 1e-9
    ids, diff, cov = node.mapper.edges()
    assert np.array_equal(ids, want["edges"][0])
    assert np.abs(diff - want["edges"][1]).max(initial=0.0) <= 1e-9
    assert len(got["maps"]) == len(want["maps"]) == len(own)
    for (gi, ginfo, gmap), (wi, winfo, wmap), (g, payload) in zip(got["maps"], want["maps"], own):
        assert gi == wi and (ginfo["width"], ginfo["height"]) == (winfo["width"], winfo["height"])
        # the grid's offset is the scans' bounding-box minimum, from the device's sin / cos: equal to the last place or so
        assert np.abs(ginfo["offset"] - g["offset"]).max() <= 1e-9
        assert np.array_equal(gmap, karto_node_port.ros_payload(g)), (name, gi)
        assert np.array_equal(gmap, wmap), (name, gi)
        assert np.abs(ginfo["offset"] - winfo["offset"]).max() <= 1e-9
    node.close()


def laser_of(c):
    return karto_node_port.laser_of(c.geometry(), c.mount, KN.node_params(c.params)[0].use_scan_range)[0]


def readings_of(c, node):
    """the readings of every scan the node processed so far, as it keeps them"""
    laser, inverted = karto_node_port.laser_of(c.geometry(), c.mount, KN.node_params(c.params)[0].use_scan_range)
    return _readings(c, node, laser, inverted)


def _readings(c, node, laser, inverted):
    want = ported(c.name)
    n = node.mapper.L.b2s_mapper_scan_count(node.mapper.h)
    rows = [i for i in range(len(want["state"])) if want["state"][i] == karto_node_port.PROCESSED][:n]
    r = c.ranges[rows][:, ::-1] if inverted else c.ranges[rows]
    return r[:, :laser.n_readings].astype(np.float64)


@pytest.mark.parametrize("name", ["throttle_3", "back_end", "interval_exact"])
def test_chunked_calls_equal_one_call(name):
    c = kc.CASES[name]
    one = device_node(c).process(c.ranges, c.stamps, c.odom)
    node = device_node(c)
    cuts = [0, 1, 7, 8, 20, len(c.ranges)]
    parts = [node.process(c.ranges[a:b], c.stamps[a:b], c.odom[a:b]) for a, b in zip(cuts, cuts[1:])]
    for k in ("state", "pose", "map_to_odom", "map_published"):
        assert np.array_equal(np.concatenate([p[k] for p in parts]), one[k]), k
    maps = [m for p in parts for m in p["maps"]]
    assert [m[0] for m in maps] == [m[0] for m in one["maps"]]
    assert all(np.array_equal(a[2], b[2]) for a, b in zip(maps, one["maps"]))


def test_node_equals_per_scan_route():
    """b2s_mapper_process_sensor per scan plus b2s_occ_grid_create_from_scans whenever the node publishes"""
    c = kc.CASES["loops_small_windows"]
    got = device_node(c).process(c.ranges, c.stamps, c.odom)
    prm, _ = KN.node_params(c.params)
    laser, inverted = karto_node_port.laser_of(c.geometry(), c.mount, prm.use_scan_range)
    prm.mapper.sequential.range_threshold = prm.mapper.loop.range_threshold = laser.range_threshold
    m = MP.Mapper(prm.mapper, laser)
    kept, maps = [], []
    for i in range(len(c.ranges)):
        od = c.odom[i]
        op = karto_node_port._mul(karto_node_port._from_row(od), (karto_node_port._rotation(karto_node_port._quat_rpy(0.0, 0.0, 0.0)),
                                                                 [0.0, 0.0, 0.0]))
        yaw = karto_node_port._yaw(karto_node_port._quaternion(op[0]))
        od = op[1]
        r = c.ranges[i][:laser.n_readings].astype(np.float64)
        ok, pose = m.process(r, (od[0], od[1], yaw), 0.0, sensor="laser")
        if ok:
            kept.append(r)
            assert np.array_equal(pose, got["pose"][i])
        if got["map_published"][i]:
            g = OG.OccupancyGrid(laser, np.array(kept), m.poses(), prm.resolution)
            maps.append(g.ros_map())
            g.close()
    assert len(maps) == len(got["maps"]) >= 2
    assert all(np.array_equal(a, b[2]) for a, b in zip(maps, got["maps"]))
    m.close()


def test_refused_process_writes_nothing():
    c = kc.CASES["standing_still"]
    node = device_node(c)
    L, S = node.L, 3
    state, pose = np.full(S, 77, np.int32), np.full((S, 3), 7.0)
    i32, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
    r = np.ascontiguousarray(c.ranges[:S])
    for args in ((S, r.ctypes.data_as(C.POINTER(C.c_float)), None), (-1, r.ctypes.data_as(C.POINTER(C.c_float)), None)):
        rc = L.b2s_karto_node_process(node.h, args[0], args[1], None, None, state.ctypes.data_as(i32),
                                      pose.ctypes.data_as(dp), None, None, KN.MAP_FN(), None)
        assert rc == 1
    assert (state == 77).all() and (pose == 7.0).all()
    got = node.process(c.ranges, c.stamps, c.odom)  # nothing was counted by the refused calls
    assert np.array_equal(got["state"], ported("standing_still")["state"])
    node.close()
