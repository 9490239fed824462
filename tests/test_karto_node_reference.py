"""lesson6's Karto SLAM node over whole recordings (CPU): the restatement oracle/karto_node_port.py (the node's logic in
Python over the library's host Mapper, the C restatement's MatchScan and occupancy grid) against the unmodified
SlamKarto (oracle/ref_lesson6.cpp), live where oracle/_ref/ is built and replayed from tests/golden/reference/
elsewhere; that every case of tests/karto_node_cases.py does what it is named for; and the refusals of
b2s_karto_node_create that need no device."""
import ctypes as C
import functools
import importlib

import numpy as np
import pytest

import karto_node_cases as kc
from oracle import karto_node_port, ref_lesson6
from reference_record import digest, recording

KN = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.karto_node")
M = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.matcher")


@functools.lru_cache(maxsize=None)
def ported(name):
    c = kc.CASES[name]
    prm, use_back_end = KN.node_params(c.params)
    node = karto_node_port.PortKartoNode(prm, c.geometry(), c.mount, kc.pose_graph() if use_back_end else None)
    out = node.process(c.ranges, c.stamps, c.odom)
    ids, diff, cov = node.mapper.edges()
    out.update(edges=(ids, diff, cov.reshape(-1, 9)), poses=node.mapper.poses(), node=node,
               loops=node.mapper.stats()["loops_closed"])
    return out


def summary(o):
    """What is compared: maps through their digests, dimensions and origins"""
    maps = o["maps"]
    return dict(state=o["state"], map_published=o["map_published"], pose=o["pose"], map_to_odom=o["map_to_odom"],
                map_scans=np.array([m[0] for m in maps], np.int32),
                map_dims=np.array([(m[1]["width"], m[1]["height"]) for m in maps], np.int32).reshape(-1, 2),
                map_origins=np.array([m[1]["offset"] for m in maps], np.float64).reshape(-1, 2),
                map_digests=[digest(m[2]) for m in maps], edge_ids=o["edges"][0], edge_diff=o["edges"][1],
                edge_cov=np.asarray(o["edges"][2]).reshape(-1, 9), poses=o["poses"])


def node_answer(c):
    solver = kc.pose_graph() if c.use_back_end else None
    return summary(ref_lesson6.run(c.params, c.fields, c.mount, c.ranges, c.stamps, c.odom, solver=solver))


@pytest.mark.parametrize("name", list(kc.CASES))
def test_port_equals_node(request, name):
    """States, published-map flags, graph edge ids and map bytes exactly; corrected poses, map_to_odom, edge pose
    differences and the final graph poses to 1e-12 (0 observed); edge covariances to 1e-9 relative."""
    c = kc.CASES[name]
    with recording(request, ref_lesson6.available()) as rec:
        want = rec.value("node", lambda: node_answer(c), inputs=(c.params, c.fields, c.mount, c.ranges, c.stamps, c.odom))
    got = summary(ported(name))
    for k in ("state", "map_published", "map_scans", "map_dims", "map_origins", "edge_ids"):
        assert np.array_equal(got[k], want[k]), (name, k)
    assert got["map_digests"] == list(want["map_digests"]), name
    for k in ("pose", "map_to_odom", "edge_diff", "poses"):
        assert np.asarray(got[k]).shape == np.asarray(want[k]).shape, (name, k)
        assert np.abs(got[k] - want[k]).max(initial=0.0) <= 1e-12, (name, k)
    assert np.allclose(got["edge_cov"], want["edge_cov"], rtol=1e-9, atol=1e-15), name


@pytest.mark.parametrize("name", list(kc.CASES))
def test_cases_cover_the_node(name):
    """Each recording exercises what its name says."""
    c, o = kc.CASES[name], ported(name)
    node, st, pub = o["node"], o["state"], o["map_published"]
    for e in c.expect:
        if e == "maps>=2":
            assert len(o["maps"]) >= 2, name
        elif e == "one_map":
            assert len(o["maps"]) == 1, name
        elif e == "map_every_processed":
            assert np.array_equal(pub, (st == karto_node_port.PROCESSED).astype(np.int32)), name
        elif e == "loops":
            assert o["loops"] > 0, name
        elif e == "near_links":
            assert len(o["edges"][0]) > len(o["poses"]) - 1 and o["loops"] == 0, name
        elif e == "throttled":
            assert (st == karto_node_port.THROTTLED).any() and (st == karto_node_port.PROCESSED).any(), name
        elif e == "no_odom":
            assert (st == karto_node_port.NO_ODOM).sum() == 5, name
        elif e == "not_moved":
            assert (st == karto_node_port.NOT_MOVED).any(), name
        elif e == "inverted":
            assert node.inverted, name
        elif e == "last_beam_dropped":
            assert node.laser.n_readings == c.ranges.shape[1] - 1, name
        elif e == "exact_interval_no_map":
            iv, last, seen = karto_node_port.duration_from_sec(c.params["map_update_interval"]), None, False
            for i in range(len(st)):
                s = (int(c.stamps[i][0]), int(c.stamps[i][1]))
                if st[i] == karto_node_port.PROCESSED and last is not None and karto_node_port.stamp_diff(s, last) == iv:
                    assert not pub[i], name
                    seen = True
                if pub[i]:
                    last = s
            assert seen and c.stamps[0][1] != 0, name
        elif e == "poses_moved":
            moved = any(not np.array_equal(a, b[:len(a)]) for a, b in zip(node.map_poses, node.map_poses[1:]))
            assert moved, name
        else:
            raise AssertionError(f"unknown expectation {e}")
    if not (c.standard_geometry or "inverted" in c.expect):
        assert node.laser.n_readings == c.ranges.shape[1] and not node.inverted, name


def _create(params, geometry, mount=(0, 0, 0, 0, 0, 0, 1.0)):
    L = KN._bind()
    h = C.c_void_p()
    m = np.array(mount, np.float64)
    rc = L.b2s_karto_node_create(C.byref(params), C.byref(geometry), m.ctypes.data_as(C.POINTER(C.c_double)), None, 0,
                                 C.byref(h))
    return rc, h


@pytest.mark.parametrize("what", ["throttle_0", "throttle_negative", "resolution_0", "fewer_ranges", "zero_quaternion",
                                  "interval_nan"])
def test_create_refusals(what):
    """Refused before any device is touched: B2S_ERR_BAD_PARAMS and no handle."""
    c = kc.CASES["defaults"]
    prm, _ = KN.node_params(c.params)
    geometry, mount = c.geometry(), (0, 0, 0, 0, 0, 0, 1.0)
    if what == "throttle_0":
        prm.throttle_scans = 0
    elif what == "throttle_negative":
        prm.throttle_scans = -2
    elif what == "resolution_0":
        prm.resolution = 0.0
    elif what == "fewer_ranges":
        geometry.n_ranges = geometry.n_ranges - 1  # m = n readings expected, one fewer carried
    elif what == "zero_quaternion":
        mount = (0, 0, 0, 0, 0, 0, 0.0)
    elif what == "interval_nan":
        prm.map_update_interval = float("nan")
    rc, h = _create(prm, geometry, mount)
    assert rc == 1 and not h.value, what


def test_create_without_device():
    if M.device_count() > 0:
        pytest.skip("a CUDA device is present")
    c = kc.CASES["standard_geometry"]
    prm, _ = KN.node_params(c.params)
    rc, h = _create(prm, c.geometry())
    assert rc == 5 and not h.value


def test_node_params_follow_init_params():
    """Absent parameters keep the defaults; three are squared; minimum_time_interval is never read."""
    d, ube = KN.node_params({})
    assert (d.throttle_scans, d.map_update_interval, d.resolution, d.use_scan_range, ube) == (1, 5.0, 0.05, 12.0, False)
    assert d.mapper.minimum_time_interval == 3600 and d.mapper.sequential.distance_variance_penalty == 0.3 * 0.3
    p, ube = KN.node_params(kc.SHIPPED_YAML)
    assert not ube and p.mapper.minimum_time_interval == 3600 and p.mapper.scan_buffer_size == 110
    assert p.mapper.loop_match_maximum_variance_coarse == 9.0
    for m in (p.mapper.sequential, p.mapper.loop):
        assert m.distance_variance_penalty == 0.5 * 0.5 and m.angle_variance_penalty == 0.1 * 0.1
        assert m.coarse_search_angle_offset == 0.349 and m.use_response_expansion == 1
    assert (p.mapper.sequential.search_size, p.mapper.loop.search_size, p.mapper.loop.resolution) == (0.3, 10.0, 0.05)
