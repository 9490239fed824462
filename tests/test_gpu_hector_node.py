"""GPU tests of b2s_hector_node_* (lesson4's HectorMappingRos over whole recordings): the handle must equal the
restatement oracle/hector_node_port.py bit for bit on every recording of hector_node_cases: poses, Hessians (the
covariance message), gate flags, kept-beam counts, pose messages, map payloads, map info, publish stamps and rebuild
flags.  Also: chunked calls equal one call, a yaw-only mount equals b2s_hector_slam_process_scans_batch, publish_map
equals the scheduled map, and refused calls write nothing."""
import ctypes as C

import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def N(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector_node")


@pytest.fixture(scope="module")
def R(pkg):
    return pkg.load("rosio")


def _geom(R, g, n):
    amin, inc, rmin, rmax = g
    return R.make_msg(amin, amin + inc * f32(n - 1), inc, rmin, rmax, np.zeros(n, np.float32))


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _assert_maps(got, want, what):
    assert len(got) == len(want), what
    for k, (g, w) in enumerate(zip(got, want)):
        assert (g["scan_index"], g["stamp"], g["rebuilt"]) == (w["scan_index"], w["stamp"], w["rebuilt"]), (what, k)
        for f in ("origin_x", "origin_y", "width", "height"):
            assert g["info"][f] == w["info"][f], (what, k, f)
        assert f32(g["info"]["resolution"]) == f32(w["info"]["resolution"]), (what, k)
        assert np.array_equal(g["payload"], w["payload"]), (what, k)


def _assert_scans(got, want, what):
    assert _same_bits(got["pose"], want["pose"]), what
    assert np.array_equal(got["map_updated"], want["map_updated"]), what
    assert np.array_equal(got["n_points"], want["n_points"]), what
    assert _same_bits(got["pose_msg"], want["pose_msg"]), what
    keep = ~cases.uninitialised_rows(want["n_points"])
    assert _same_bits(got["cov"][keep], want["cov"][keep]), what
    assert not got["cov"][~keep].any(), what  # the handle's zeros where the node reads an uninitialised matrix


def _node(N, R, c):
    return N.HectorNode(N.node_params(c["params"]), _geom(R, c["geometry"], c["ranges"].shape[1]), c["mount"])


def _port(N, c):
    p = N.node_params(c["params"])
    d = {f: getattr(p, f) for f, _ in N.HectorNodeParams._fields_}
    return P.HectorNodePort(d, c["geometry"], c["mount"])


CASES = cases.cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_handle_equals_the_port(N, R, name):
    c = CASES[name]
    g = _node(N, R, c)
    got = g.process(c["ranges"], c["stamps"])
    port = _port(N, c)
    want = port.process(c["ranges"], c["stamps"])
    _assert_scans(got, want, name)
    _assert_maps(got["maps"], want["maps"], name)
    assert len(got["maps"]) >= 1 and got["maps"][0]["rebuilt"] and (got["maps"][0]["payload"] == -1).all()
    # the processor getter serves the node: level 0 now equals the port's final grid as a payload
    final = port.publish_map((0, 0))["payload"]
    assert np.array_equal(g.level_ros(0), final), name
    if name == "rare_gate":
        assert got["map_updated"].sum() == 1 and not any(m["rebuilt"] for m in got["maps"][2:])
    if name == "empty_scans":
        assert (got["n_points"][[0, 1, 5, 6]] == 0).all()
    port.close(), g.close()


@pytest.mark.parametrize("cuts", [(1, 4, 7), (3,), (2, 5, 6, 9)])
def test_chunked_calls_equal_one_call(N, R, cuts):
    c = CASES["bad_ranges"]  # publishes before every other scan: the cuts fall on and off publish points
    a = _node(N, R, c)
    whole = a.process(c["ranges"], c["stamps"])
    b = _node(N, R, c)
    parts = []
    edges = (0,) + cuts + (len(c["ranges"]),)
    for lo, hi in zip(edges[:-1], edges[1:]):
        parts.append(b.process(c["ranges"][lo:hi], c["stamps"][lo:hi]))
    joined = {k: np.concatenate([p[k] for p in parts]) for k in ("pose", "pose_msg", "cov", "map_updated", "n_points")}
    for k in joined:
        assert _same_bits(joined[k], whole[k]), (cuts, k)
    _assert_maps([m for p in parts for m in p["maps"]], whole["maps"], cuts)
    a.close(), b.close()


def test_yaw_only_mount_equals_the_processor_route(pkg, N, R):
    """Identity basis with a translation and thresholds whose float and double squares agree (0.25, 30): the node's
    conversion keeps the beams b2s_hector_slam_process_scans_batch keeps, and the poses and flags are the same."""
    H = pkg.load("hector")
    r = cases.walk(21, 10)
    st = cases.stamps_at(3, 0, 25_000_000, 10)
    lb = (0.125, -0.0625, 0.25)
    params = dict(cases.SMALL, laser_min_dist=0.25, map_update_distance_thresh=0.1, map_update_angle_thresh=0.9)
    c = dict(params=params, mount=cases.mount(*lb), geometry=cases.GEOMETRY, ranges=r, stamps=st)
    g = _node(N, R, c)
    got = g.process(r, st)
    h = H.HectorSlam(resolution=0.05, size_x=512, size_y=512, levels=3, min_dist=0.1, min_angle=0.9, batch=1,
                     max_points=r.shape[1])
    geom = _geom(R, cases.GEOMETRY, r.shape[1])
    res, covs, kept = h.process_scans_batch(geom, [r], R.hector_scan_filter(laser_in_base=lb + (0.0,), min_dist=0.25),
                                            first_hints=np.zeros((1, 3), np.float32))
    assert _same_bits(got["pose"], res[0][0]) and np.array_equal(got["map_updated"], res[0][1])
    assert np.array_equal(got["n_points"], kept[0])
    assert _same_bits(got["cov"][-1], np.array(P.pose_message(res[0][0][-1], covs[0])[1]))
    g.close(), h.close()


def test_publish_map_equals_the_scheduled_map(N, R):
    c = CASES["schedule_gaps"]
    a = _node(N, R, c)
    whole = a.process(c["ranges"], c["stamps"])
    k = next(m for m in whole["maps"] if m["scan_index"] > 0)
    b = _node(N, R, c)
    b.process(c["ranges"][:k["scan_index"]], c["stamps"][:k["scan_index"]])
    m = b.publish_map(k["stamp"])
    assert (m["scan_index"], m["stamp"], m["rebuilt"]) == (k["scan_index"], k["stamp"], k["rebuilt"])
    assert m["info"] == k["info"] and np.array_equal(m["payload"], k["payload"])
    again = b.publish_map(k["stamp"])  # the gate: nothing changed since
    assert not again["rebuilt"] and np.array_equal(again["payload"], k["payload"])
    a.close(), b.close()


def test_refused_calls_write_nothing(pkg, N, R):
    abi = pkg.abi
    c = CASES["empty_scans"]
    g = _node(N, R, c)
    g.process(c["ranges"][:3], c["stamps"][:3])
    L = g.L
    S, n = 2, c["ranges"].shape[1]
    pose = np.full((S, 3), 7.0, np.float32)
    msg, cov = np.full((S, 7), 7.0), np.full((S, 36), 7.0)
    upd, kept = np.full(S, 7, np.int32), np.full(S, 7, np.int32)
    r = np.ascontiguousarray(c["ranges"][3:5])
    st = np.ascontiguousarray(c["stamps"][3:5])
    fp, dp, ip = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
    calls = []

    def cb(*a):
        calls.append(a)
    fn = N.MAP_FN(cb)

    def raw(count, rr, ss):
        return L.b2s_hector_node_process(g.h, count, rr.ctypes.data_as(fp) if rr is not None else None,
                                         ss.ctypes.data_as(C.POINTER(C.c_uint32)) if ss is not None else None,
                                         pose.ctypes.data_as(fp), msg.ctypes.data_as(dp), cov.ctypes.data_as(dp),
                                         upd.ctypes.data_as(ip), kept.ctypes.data_as(ip), fn, None)
    assert raw(-1, r, st) == abi.B2S_ERR_BAD_PARAMS
    assert raw(S, None, st) == abi.B2S_ERR_BAD_PARAMS
    assert raw(S, r, None) == abi.B2S_ERR_BAD_PARAMS
    assert (pose == 7).all() and (msg == 7).all() and (cov == 7).all() and (upd == 7).all() and (kept == 7).all()
    assert not calls
    # the node goes on as if nothing had been refused
    ref = _node(N, R, c)
    want = ref.process(c["ranges"], c["stamps"])
    rest = g.process(c["ranges"][3:], c["stamps"][3:])
    assert _same_bits(rest["pose"], want["pose"][3:])
    assert [m["scan_index"] for m in rest["maps"]] == [m["scan_index"] for m in want["maps"] if m["scan_index"] >= 3]
    g.close(), ref.close()


def test_create_refusals(pkg, N, R):
    abi = pkg.abi
    L = N._bind()
    geom = _geom(R, cases.GEOMETRY, 1081)
    h = C.c_void_p()
    dp = C.POINTER(C.c_double)

    def create(params=None, g=geom, mount=cases.mount()):
        p = params if params is not None else N.node_params()
        m = np.ascontiguousarray(mount, np.float64)
        return L.b2s_hector_node_create(C.byref(p), C.byref(g) if g is not None else None, m.ctypes.data_as(dp), 0,
                                        C.byref(h))
    assert create(g=None) == abi.B2S_ERR_BAD_PARAMS
    assert create(mount=(0, 0, 0, 0, 0, 0, 0)) == abi.B2S_ERR_BAD_PARAMS
    assert create(mount=(0, 0, np.nan, 0, 0, 0, 1)) == abi.B2S_ERR_BAD_PARAMS
    for key, v in [("map_resolution", 0.0), ("map_size", 0), ("map_pub_period", 0.0), ("map_pub_period", np.inf),
                   ("map_pub_period", 1e-12), ("map_pub_period", 3e9)]:
        assert create(N.node_params({key: v})) == abi.B2S_ERR_BAD_PARAMS, key
    zero_inc = R.make_msg(f32(0), f32(1), f32(0), f32(0.1), f32(30), np.zeros(10, np.float32))
    assert create(g=zero_inc) == abi.B2S_ERR_BAD_PARAMS
    assert create(g=_geom(R, cases.GEOMETRY, 4097)) == abi.B2S_ERR_TOO_LARGE
    assert not h.value
