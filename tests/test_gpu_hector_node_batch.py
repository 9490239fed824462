"""GPU tests of b2s_hector_node_create_batch / _process_batch / _publish_map_of: several lesson4 HectorMappingRos nodes
in one handle.  Every node must equal, bit for bit, its own single-node handle (and the restatement
oracle/hector_node_port.py where a case has one): poses, pose messages, covariances, gate flags, kept-beam counts and
every map's payload, info, stamp, scan_index and rebuilt flag.  Also: chunked calls (some nodes without scans) equal
one call, more nodes than resident CTAs, the on-demand publish of one node, and refusals that write and change
nothing."""
import ctypes as C

import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P
from test_gpu_hector_node import _assert_maps, _assert_scans, _geom, _node, _port, _same_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
CASES = cases.cases()
SHARED = ["yaw_pi", "upside_down", "pitched_z_window", "bad_ranges", "empty_scans", "schedule_gaps", "short_period"]


@pytest.fixture(scope="module")
def N(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector_node")


@pytest.fixture(scope="module")
def R(pkg):
    return pkg.load("rosio")


def _batch(N, R, cs):
    return N.HectorNodeBatch([N.node_params(c["params"]) for c in cs], _geom(R, cs[0]["geometry"], cs[0]["ranges"].shape[1]),
                             [c["mount"] for c in cs])


def _single(N, R, c):
    g = _node(N, R, c)
    out = g.process(c["ranges"], c["stamps"])
    g.close()
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_batch_of_one_equals_the_node(N, R, name):
    c = CASES[name]
    h = _batch(N, R, [c])
    (got,) = h.process([c["ranges"]], [c["stamps"]])
    want = _single(N, R, c)
    _assert_scans(got, want, name)
    _assert_maps(got["maps"], want["maps"], name)
    h.close()


def test_shared_processor_cases_in_one_batch(N, R):
    cs = [CASES[n] for n in SHARED]
    h = _batch(N, R, cs)
    order = []
    got = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs], on_map=None)
    for b, (name, c) in enumerate(zip(SHARED, cs)):
        port = _port(N, c)
        want = port.process(c["ranges"], c["stamps"])
        _assert_scans(got[b], want, name)
        _assert_maps(got[b]["maps"], want["maps"], name)
        _assert_maps(got[b]["maps"], _single(N, R, c)["maps"], name)
        assert np.array_equal(h.level_ros(b), port.publish_map((0, 0))["payload"]), name
        port.close()
    # the order across nodes: part by part, nodes ascending inside a part
    h2 = _batch(N, R, cs)
    h2.process([c["ranges"] for c in cs], [c["stamps"] for c in cs], on_map=lambda b, m: order.append((b, m["scan_index"])))
    per_node = {b: [m["scan_index"] for m in got[b]["maps"]] for b in range(len(cs))}
    rank = {}  # the part of node b's j-th map is j + 1 (a node's first map opens part 1 or is at scan 0 of part 1)
    for b, idx in per_node.items():
        for j, s in enumerate(idx):
            rank[(b, s)] = j
    assert order == sorted(order, key=lambda t: (rank[t], t[0]))
    h.close(), h2.close()


def _walks(seed, B, max_len=60):
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        n = int(rng.integers(0, max_len + 1))
        period = float(rng.choice([0.025, 0.05, 0.1, 0.3, 2.0]))
        m = cases.mount(float(rng.uniform(-0.1, 0.1)), float(rng.uniform(-0.1, 0.1)), float(rng.uniform(0.0, 0.4)),
                        yaw=float(rng.uniform(-3.1, 3.1)), roll=float(rng.choice([0.0, np.pi])))
        r = cases.walk(1000 + seed * 1000 + b, max(n, 1))[:n]
        st = cases.stamps_at(int(rng.integers(1, 100)), int(rng.integers(0, 1_000_000_000)), 25_000_000, n,
                             gaps=((int(rng.integers(0, max(n, 1))), int(rng.integers(0, 3_000_000_000))),))
        out.append(dict(params=dict(cases.SMALL, map_pub_period=period,
                                    laser_z_min_value=float(rng.choice([-1.0, -0.3])),
                                    laser_max_dist=float(rng.choice([30.0, 12.0]))),
                        mount=m, geometry=cases.GEOMETRY, ranges=r, stamps=st.reshape(n, 2)))
    return out


def _each_equals_single(N, R, cs, got):
    for b, c in enumerate(cs):
        if len(c["stamps"]) == 0:
            assert len(got[b]["pose"]) == 0 and not got[b]["maps"]
            continue
        want = _single(N, R, c)
        _assert_scans(got[b], want, b)
        _assert_maps(got[b]["maps"], want["maps"], b)


def test_ragged_batch_and_chunked_calls(N, R):
    cs = _walks(7, 40)
    h = _batch(N, R, cs)
    whole = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    _each_equals_single(N, R, cs, whole)
    # three calls, each node cut at its own points (some calls give a node no scans)
    rng = np.random.default_rng(3)
    edges = [np.sort(np.concatenate([[0], rng.integers(0, len(c["stamps"]) + 1, 2), [len(c["stamps"])]])) for c in cs]
    h2 = _batch(N, R, cs)
    parts = [h2.process([c["ranges"][e[k]:e[k + 1]] for c, e in zip(cs, edges)],
                        [c["stamps"][e[k]:e[k + 1]] for c, e in zip(cs, edges)]) for k in range(3)]
    for b in range(len(cs)):
        for key in ("pose", "pose_msg", "cov", "map_updated", "n_points"):
            assert _same_bits(np.concatenate([p[b][key] for p in parts]), whole[b][key]), (b, key)
        _assert_maps([m for p in parts for m in p[b]["maps"]], whole[b]["maps"], b)
    h.close(), h2.close()


def test_more_nodes_than_resident_ctas(N, R):
    cs = _walks(11, 269, max_len=24)
    h = _batch(N, R, cs)
    got = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    _each_equals_single(N, R, cs, got)
    h.close()


def test_publish_map_of_one_node(N, R):
    cs = [CASES[n] for n in SHARED]
    h = _batch(N, R, cs)
    b = SHARED.index("schedule_gaps")
    whole = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    k = next(m for m in whole[b]["maps"] if m["scan_index"] > 0)
    h2 = _batch(N, R, cs)
    h2.process([c["ranges"][:k["scan_index"]] if j == b else c["ranges"] for j, c in enumerate(cs)],
               [c["stamps"][:k["scan_index"]] if j == b else c["stamps"] for j, c in enumerate(cs)])
    m = h2.publish_map(b, k["stamp"])
    assert (m["scan_index"], m["stamp"], m["rebuilt"]) == (k["scan_index"], k["stamp"], k["rebuilt"])
    assert m["info"] == k["info"] and np.array_equal(m["payload"], k["payload"])
    assert not h2.publish_map(b, k["stamp"])["rebuilt"]  # node b's gate
    # the other nodes' gates did not move: their final publish equals that of a handle never asked for node b's map
    for j in range(len(cs)):
        if j != b:
            assert h2.publish_map(j, (0, 0))["rebuilt"] == h.publish_map(j, (0, 0))["rebuilt"], j
    h.close(), h2.close()


def test_refusals(pkg, N, R):
    abi = pkg.abi
    L = N._bind()
    cs = [CASES[n] for n in SHARED[:3]]
    geom = _geom(R, cases.GEOMETRY, 1081)
    hh = C.c_void_p()
    dp = C.POINTER(C.c_double)

    def create(ps, mounts):
        arr = (N.HectorNodeParams * len(ps))(*ps)
        m = np.ascontiguousarray(mounts, np.float64)
        return L.b2s_hector_node_create_batch(len(ps), arr, C.byref(geom), m.ctypes.data_as(dp), 0, C.byref(hh))
    ps = [N.node_params(c["params"]) for c in cs]
    mounts = [c["mount"] for c in cs]
    for key, v in [("map_size", 1024), ("map_resolution", 0.1), ("update_factor_free", 0.3),
                   ("map_update_angle_thresh", 0.5), ("map_multi_res_levels", 2)]:
        bad = list(ps)
        bad[2] = N.node_params(dict(cs[2]["params"], **{key: v}))
        assert create(bad, mounts) == abi.B2S_ERR_BAD_PARAMS, key
    assert create(ps, mounts[:2] + [(0, 0, 0, 0, 0, 0, 0)]) == abi.B2S_ERR_BAD_PARAMS
    assert b"node 2" in L.b2s_last_error()
    assert not hh.value
    # a batch with different periods, z windows and range limits is accepted
    assert create(ps, mounts) == abi.B2S_OK
    L.b2s_hector_node_destroy(hh)

    h = _batch(N, R, cs)
    first = h.process([c["ranges"][:3] for c in cs], [c["stamps"][:3] for c in cs])
    S = 2 * len(cs)
    pose = np.full((S, 3), 7.0, np.float32)
    msg, cov = np.full((S, 7), 7.0), np.full((S, 36), 7.0)
    upd, kept = np.full(S, 7, np.int32), np.full(S, 7, np.int32)
    r = np.ascontiguousarray(np.concatenate([c["ranges"][3:5] for c in cs]))
    st = np.ascontiguousarray(np.concatenate([c["stamps"][3:5] for c in cs]))
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    calls = []
    fn = N.BATCH_MAP_FN(lambda *a: calls.append(a))

    def raw(counts, rr, ss):
        cnt = np.ascontiguousarray(counts, np.int32) if counts is not None else None
        return L.b2s_hector_node_process_batch(h.h, cnt.ctypes.data_as(ip) if cnt is not None else None,
                                               rr.ctypes.data_as(fp) if rr is not None else None,
                                               ss.ctypes.data_as(C.POINTER(C.c_uint32)) if ss is not None else None,
                                               pose.ctypes.data_as(fp), msg.ctypes.data_as(dp), cov.ctypes.data_as(dp),
                                               upd.ctypes.data_as(ip), kept.ctypes.data_as(ip), fn, None)
    assert raw([2, -1, 2], r, st) == abi.B2S_ERR_BAD_PARAMS
    assert raw(None, r, st) == abi.B2S_ERR_BAD_PARAMS
    assert raw([2, 2, 2], None, st) == abi.B2S_ERR_BAD_PARAMS
    assert raw([2, 2, 2], r, None) == abi.B2S_ERR_BAD_PARAMS
    assert raw([2, (1 << 20) - 1, 2], r, st) == abi.B2S_ERR_TOO_LARGE
    assert (pose == 7).all() and (msg == 7).all() and (cov == 7).all() and (upd == 7).all() and (kept == 7).all()
    assert not calls
    # the single-node entry points refuse a handle of several nodes
    one = (C.c_uint32 * 2)(0, 0)
    assert L.b2s_hector_node_publish_map(h.h, one, N.MAP_FN(lambda *a: None), None) == abi.B2S_ERR_BAD_PARAMS
    assert L.b2s_hector_node_publish_map_of(h.h, 3, one, fn, None) == abi.B2S_ERR_BAD_PARAMS
    # the handle goes on as a fresh one would
    rest = h.process([c["ranges"][3:] for c in cs], [c["stamps"][3:] for c in cs])
    ref = _batch(N, R, cs)
    want = ref.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    for b in range(len(cs)):
        for key in ("pose", "pose_msg", "cov", "map_updated", "n_points"):
            assert _same_bits(np.concatenate([first[b][key], rest[b][key]]), want[b][key]), (b, key)
        _assert_maps(first[b]["maps"] + rest[b]["maps"], want[b]["maps"], b)
    h.close(), ref.close()
