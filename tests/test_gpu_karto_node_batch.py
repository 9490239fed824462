"""Many lesson6 Karto SLAM nodes in one handle (b2s_karto_node_create_batch / _process_batch) against their own
single-node handles (b2s_karto_node_create), which tests/test_gpu_karto_node.py pins to the restatement: every node
equals its single handle bit for bit in states, published flags, poses, map_to_odom, graph edges, b2s_mapper_stats and
every map (scan index, info, payload).  Also: 132 ragged recordings at once, chunked calls, the batched map build
against b2s_occ_grid_create_from_scans, refusals, and that no thread outlives a call."""
import ctypes as C
import functools
import importlib
import math
import os

import numpy as np
import pytest

import karto_node_cases as kc
from oracle import karto_node_port

pytestmark = pytest.mark.gpu
KN = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.karto_node")
OG = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.occgrid")
MP = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.mapper")

# the identity-mount cases with SMALL's matcher windows: one laser, one pair of matchers, different throttles, intervals,
# back ends and lengths
SMALL_GROUP = ["loops_small_windows", "throttle_3", "interval_0", "interval_1e6", "interval_exact", "standing_still",
               "odom_failures", "bad_readings", "back_end"]


def solver_for(params):
    return kc.pose_graph() if params.get("use_back_end") else None


def run_single(params, geometry, mount, ranges, stamps, odom, cuts=None):
    prm, _ = KN.node_params(params)
    node = KN.KartoNode(prm, geometry, mount, solver_for(params))
    got = node.process(ranges, stamps, odom)
    got["edges"] = node.mapper.edges()
    got["stats"] = node.mapper.stats()
    got["poses_now"] = node.mapper.poses()
    node.close()
    return got


@functools.lru_cache(maxsize=None)
def single_case(name):
    c = kc.CASES[name]
    return run_single(c.params, c.geometry(), c.mount, c.ranges, c.stamps, c.odom)


def run_fleet(params_list, geometry, mounts, ranges, stamps, odom, order=None):
    prms = [KN.node_params(p)[0] for p in params_list]
    fleet = KN.KartoNodeBatch(prms, geometry, mounts, [solver_for(p) for p in params_list])
    got = fleet.process(ranges, stamps, odom, on_map=(lambda b, i, info, data: order.append((b, i))) if order is not None
                        else None)
    for b, g in enumerate(got):
        g["edges"] = fleet.mapper(b).edges()
        g["stats"] = fleet.mapper(b).stats()
        g["poses_now"] = fleet.mapper(b).poses()
    timing = fleet.last_timing()
    fleet.close()
    return got, timing


def assert_same_node(got, want, who, maps="all"):
    for k in ("state", "map_published", "pose", "map_to_odom"):
        assert np.array_equal(got[k], want[k]), (who, k)
    for k in range(3):
        assert np.array_equal(got["edges"][k], want["edges"][k]), (who, "edges", k)
    assert got["stats"] == want["stats"], who
    assert np.array_equal(got["poses_now"], want["poses_now"]), who
    assert len(got["maps"]) == len(want["maps"]), who
    pairs = list(zip(got["maps"], want["maps"]))
    if maps == "last":
        pairs = pairs[-1:]
    for (gi, ginfo, gmap), (wi, winfo, wmap) in pairs:
        assert gi == wi, who
        assert ginfo.keys() == winfo.keys()
        for key in ginfo:
            assert np.array_equal(ginfo[key], winfo[key]), (who, gi, key)
        assert np.array_equal(gmap, wmap), (who, gi)


def test_identity_mount_group_equals_single_handles():
    cs = [kc.CASES[n] for n in SMALL_GROUP]
    g0 = cs[0].geometry()
    order_a, order_b = [], []
    got, _ = run_fleet([c.params for c in cs], g0, [c.mount for c in cs], [c.ranges for c in cs],
                       [c.stamps for c in cs], [c.odom for c in cs], order_a)
    for c, g in zip(cs, got):
        assert_same_node(g, single_case(c.name), c.name)
        assert [m[0] for m in g["maps"]] == [i for b, i in order_a if b == cs.index(c)]
    assert any(len(g["maps"]) >= 2 for g in got)
    # the same call again: the same interleaving of maps across nodes
    run_fleet([c.params for c in cs], g0, [c.mount for c in cs], [c.ranges for c in cs], [c.stamps for c in cs],
              [c.odom for c in cs], order_b)
    assert order_a == order_b


def test_mounts_that_give_one_laser_share_a_handle():
    """mount_upside_down and the same mount 0.3 m higher: one laser, different mounts"""
    c = kc.CASES["mount_upside_down"]
    higher = (c.mount[0], c.mount[1], c.mount[2] + 0.3) + tuple(c.mount[3:])
    half = len(c.ranges) // 2
    rs, ss, os_ = [c.ranges, c.ranges[:half]], [c.stamps, c.stamps[:half]], [c.odom, c.odom[:half]]
    got, _ = run_fleet([c.params, dict(c.params, throttle_scans=2)], c.geometry(), [c.mount, higher], rs, ss, os_)
    assert_same_node(got[0], single_case(c.name), c.name)
    want = run_single(dict(c.params, throttle_scans=2), c.geometry(), higher, rs[1], ss[1], os_[1])
    assert_same_node(got[1], want, "higher")


def scale_recordings(B=132):
    """ragged recordings: prefixes of the SMALL group's recordings (a node's run is causal, so a prefix of a good run
    is a good run), with that case's throttle and back end, every third node at full length (the back_end and
    loops_small_windows nodes then close loops), the map intervals, resolutions and stamps varied"""
    rng = np.random.default_rng(132)
    params, recs = [], []
    for b in range(B):
        c = kc.CASES[SMALL_GROUP[b % len(SMALL_GROUP)]]
        S = len(c.ranges) if b % 3 == 0 else int(rng.integers(1, len(c.ranges) + 1))
        p = dict(c.params, map_update_interval=(0.0, 0.5, 1.0, 2.5)[b % 4], resolution=(0.05, 0.1, 0.03)[b % 3])
        stamps = c.stamps[:S].astype(np.int64)
        stamps[:, 0] += b
        recs.append((c.ranges[:S], stamps.astype(np.uint32), c.odom[:S]))
        params.append(p)
    return params, recs


def test_many_ragged_recordings_equal_single_handles():
    params, recs = scale_recordings()
    B = len(params)
    geom = kc.CASES["loops_small_windows"].geometry()
    ident = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    got, timing = run_fleet(params, geom, [ident] * B, [r[0] for r in recs], [r[1] for r in recs],
                            [r[2] for r in recs])
    assert timing["rounds"] > 0 and timing["maps"] > 0
    full = set(range(0, B, 8)) | {1, 2, 3}
    assert len(full) >= 16
    loops = 0
    for b in range(B):
        want = run_single(params[b], geom, ident, *recs[b])
        assert_same_node(got[b], want, b, maps="all" if b in full else "last")
        loops += want["stats"]["loops_closed"]
    assert loops > 0


def test_chunked_calls_equal_one_call():
    cs = [kc.CASES[n] for n in ["throttle_3", "back_end", "interval_exact", "standing_still"]]
    one, _ = run_fleet([c.params for c in cs], cs[0].geometry(), [c.mount for c in cs], [c.ranges for c in cs],
                       [c.stamps for c in cs], [c.odom for c in cs])
    prms = [KN.node_params(c.params)[0] for c in cs]
    fleet = KN.KartoNodeBatch(prms, cs[0].geometry(), [c.mount for c in cs], [solver_for(c.params) for c in cs])
    cuts = [[0, 0, 5, 5, 20, 45], [0, 1, 1, 40, 41, 80], [0, 30, 30, 30, 30, 30], [0, 7, 8, 9, 10, 20]]
    parts = []
    for k in range(len(cuts[0]) - 1):
        sl = [slice(cuts[b][k], cuts[b][k + 1]) for b in range(len(cs))]
        parts.append(fleet.process([c.ranges[s] for c, s in zip(cs, sl)], [c.stamps[s] for c, s in zip(cs, sl)],
                                   [c.odom[s] for c, s in zip(cs, sl)]))
    for b in range(len(cs)):
        for k in ("state", "pose", "map_to_odom", "map_published"):
            assert np.array_equal(np.concatenate([p[b][k] for p in parts]), one[b][k]), (b, k)
        maps = [m for p in parts for m in p[b]["maps"]]
        assert [m[0] for m in maps] == [m[0] for m in one[b]["maps"]]
        assert all(np.array_equal(x[2], y[2]) for x, y in zip(maps, one[b]["maps"]))
        assert np.array_equal(fleet.mapper(b).poses(), one[b]["poses_now"])
    fleet.close()


def test_batched_map_build_equals_single_grid_builds():
    c = kc.CASES["loops_small_windows"]
    laser, _ = karto_node_port.laser_of(c.geometry(), c.mount, 9.25)
    rng = np.random.default_rng(5)
    r = c.ranges[:, :laser.n_readings]
    poses = np.stack([rng.uniform(-1, 1, len(r)), rng.uniform(-1, 1, len(r)), rng.uniform(-3, 3, len(r))], 1)
    invalid = np.full((3, laser.n_readings), np.nan, np.float32)
    invalid[1] = 0.01   # below range_min
    invalid[2] = 50.0   # beyond range_max
    grids = [(r[:40], poses[:40], 0.05),       # a large grid
             (r[40:41], poses[40:41], 0.5),    # a small, coarse one
             (invalid, poses[:3], 0.05),       # all readings invalid: the box is the sensor positions
             (r[:0], poses[:0], 0.05),         # no scans: no box, no map
             (r[41:60], poses[41:60] * 3.0, 0.025),
             (r[60:61], poses[60:61], 0.1)]
    got = OG.create_from_scans_batch(laser, [g[0] for g in grids], [g[1] for g in grids], [g[2] for g in grids])
    assert got[3] is None
    for k, (rr, pp, res) in enumerate(grids):
        if len(rr) == 0:
            continue
        g = OG.OccupancyGrid(laser, rr.astype(np.float64), pp, res)
        info = g.L.b2s_occ_grid_info_get
        want_info = KN.abi.OccGridInfo()
        OG.check(info(g.h, C.byref(want_info)))
        ginfo, payload = got[k]
        assert (ginfo["width"], ginfo["height"], ginfo["width_step"], ginfo["data_size"]) == \
            (want_info.width, want_info.height, want_info.width_step, want_info.data_size), k
        assert np.array_equal(ginfo["offset"], np.array(want_info.offset[:])), k
        assert ginfo["cell_visits"] == want_info.cell_visits, k
        assert np.array_equal(payload, g.ros_map()), k
        g.close()
    assert got[0][0]["width"] > 5 * max(got[1][0]["width"], 1)


def _params(**kw):
    p = dict(kc.SMALL)
    p.update(kw)
    return KN.node_params(p)[0]


def test_refusals():
    c = kc.CASES["throttle_3"]
    geom = c.geometry()
    L = KN._bind()
    ident = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)

    def create(prms, mounts):
        h = C.c_void_p()
        arr = (KN.KartoNodeParams * len(prms))(*prms)
        m = np.ascontiguousarray(mounts, np.float64)
        rc = L.b2s_karto_node_create_batch(len(prms), arr, C.byref(geom), m.ctypes.data_as(C.POINTER(C.c_double)), None,
                                           0, C.byref(h))
        if h.value:
            L.b2s_karto_node_destroy(h)
        return rc, L.b2s_last_error().decode() if rc else ""

    # a laser that differs: offset, range threshold, upside-down flag
    for prms, mounts in (([_params(), _params()], [ident, (0.1, 0, 0, 0, 0, 0, 1)]),
                         ([_params(), _params(use_scan_range=8.0)], [ident, ident]),
                         ([_params(), _params(), _params()], [ident, ident, (0, 0, 0) + kc.quat_rpy(math.pi, 0, 0)])):
        rc, msg = create(prms, mounts)
        assert rc == 1 and "node %d" % (len(prms) - 1) in msg and "laser" in msg, msg
    # matcher parameters that differ
    rc, msg = create([_params(), _params(correlation_search_space_dimension=0.6)], [ident, ident])
    assert rc == 1 and "node 1" in msg and "matcher" in msg, msg
    rc, msg = create([_params(), _params(loop_search_space_resolution=0.1)], [ident, ident])
    assert rc == 1 and "node 1" in msg, msg
    # a node's own refusal names it
    rc, msg = create([_params(), _params(), _params(throttle_scans=0)], [ident] * 3)
    assert rc == 1 and "node 2" in msg and "throttle_scans" in msg, msg
    # host-only fields may differ
    rc, _ = create([_params(), _params(scan_buffer_size=5, do_loop_closing=False, minimum_travel_distance=0.5)],
                   [ident, ident])
    assert rc == 0
    # the node limit
    rc, msg = create([_params()] * 1025, [ident] * 1025)
    assert rc == 7, msg
    rc, _ = create([], np.zeros((0, 7)))
    assert rc == 1

    fleet = KN.KartoNodeBatch([_params(), _params(throttle_scans=3)], geom, [ident, ident])
    assert L.b2s_karto_node_mapper(fleet.h) is None
    assert L.b2s_karto_node_mapper_of(fleet.h, 2) is None and L.b2s_karto_node_mapper_of(fleet.h, -1) is None
    S = 4
    state, pose = np.full(2 * S, 77, np.int32), np.full((2 * S, 3), 7.0)
    i32, dp, fp = C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_float)
    r = np.ascontiguousarray(np.concatenate([c.ranges[:S]] * 2))
    st = np.ascontiguousarray(np.concatenate([c.stamps[:S]] * 2))
    od = np.ascontiguousarray(np.concatenate([c.odom[:S]] * 2))
    assert L.b2s_karto_node_process(fleet.h, S, r.ctypes.data_as(fp), st.ctypes.data_as(C.POINTER(C.c_uint32)),
                                    od.ctypes.data_as(dp), state.ctypes.data_as(i32), None, None, None, KN.MAP_FN(),
                                    None) == 1
    for counts, rp, sp, op in (((S, -1), r, st, od), ((S, S), None, st, od), ((S, S), r, None, od), ((S, S), r, st, None)):
        cnt = np.array(counts, np.int32)
        rc = L.b2s_karto_node_process_batch(fleet.h, cnt.ctypes.data_as(i32), rp.ctypes.data_as(fp) if rp is not None else None,
                                            sp.ctypes.data_as(C.POINTER(C.c_uint32)) if sp is not None else None,
                                            op.ctypes.data_as(dp) if op is not None else None, state.ctypes.data_as(i32),
                                            pose.ctypes.data_as(dp), None, None, KN.BATCH_MAP_FN(), None)
        assert rc == 1
    assert L.b2s_karto_node_process_batch(fleet.h, None, None, None, None, None, None, None, None, KN.BATCH_MAP_FN(),
                                          None) == 1
    assert (state == 77).all() and (pose == 7.0).all()
    # nothing was counted by the refused calls
    got = fleet.process([c.ranges, c.ranges], [c.stamps, c.stamps], [c.odom, c.odom])
    want = single_case("throttle_3")
    assert np.array_equal(got[1]["state"], want["state"]) and np.array_equal(got[1]["pose"], want["pose"])
    fleet.close()


def test_no_thread_outlives_a_call():
    cs = [kc.CASES[n] for n in ["interval_0", "interval_exact", "standing_still"]]
    prms = [KN.node_params(c.params)[0] for c in cs]
    fleet = KN.KartoNodeBatch(prms, cs[0].geometry(), [c.mount for c in cs])

    def part(a, b):
        return fleet.process([c.ranges[a:b] for c in cs], [c.stamps[a:b] for c in cs], [c.odom[a:b] for c in cs])

    part(0, 5)  # warm-up: the CUDA runtime's own threads start here
    before = len(os.listdir("/proc/self/task"))
    part(5, 12)
    part(12, 20)
    assert len(os.listdir("/proc/self/task")) == before
    fleet.close()
