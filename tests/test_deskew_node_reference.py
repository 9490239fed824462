"""lesson5's whole de-skew node over recordings (CPU): the C restatement of its callbacks, queues and per-scan
correction (oracle/deskew_node_oracle.c) against the unmodified node (oracle/ref_lesson5.cpp), live where oracle/_ref/
is built and replayed from tests/golden/reference/ elsewhere; and the refusals of b2s_lidar_undistortion_node, which
need no device.

The node sees, at each scan callback, only the number of IMU and odometry messages delivered so far
(tests/deskew_node_cases.py turns a recording with those counts into the stream the node is fed).  Its output on the
scans the restatement calls undefined (its IMU integration reads imu_time_[-1] or passes its table) is not compared."""
import ctypes as C
import importlib

import numpy as np
import pytest

import deskew_node_cases as nc
from oracle import ref_lesson5

DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")


@pytest.fixture(scope="module")
def answers():
    return nc.node_answers(ref_lesson5.available())


@pytest.mark.parametrize("name", list(nc.STREAMS))
def test_restatement_equals_node(answers, name):
    """The scans the node publishes, every cloud bit for bit, and the state it computed each from: scan times, imu_last
    and the IMU table, odometry times, the getRPY poses and the increment."""
    rec, flags, callbacks, pubs = answers[name]
    got = nc.restated(rec, flags, tables=True)
    S, n = rec["ranges"].shape
    stamps = [(int(s["sec"]), int(s["nsec"])) for s in rec["scans"]]
    node_rows = [stamps.index(tuple(int(x) for x in p["stamp"])) for p in pubs]
    fed = S if callbacks is None else callbacks
    published = [j for j in range(fed - 1) if got["status"][j] == DS.PUBLISHED]
    undefined = [j for j in range(fed - 1) if got["status"][j] == DS.UNDEFINED]
    assert set(published) <= set(node_rows) <= set(published) | set(undefined), (name, node_rows, list(got["status"]))
    assert all(got["status"][j] not in (DS.PUBLISHED, DS.UNDEFINED) for j in range(fed - 1) if j not in node_rows
               and j not in undefined)
    for j, p in zip(node_rows, pubs):
        if j in undefined:
            continue
        st = got["state"][j]
        assert nc.same(got["xyz"][j], p["xyz"]), f"{name}: scan {j}'s cloud differs from the node's"
        assert st["time_start"] == p["times"][0] and st["time_start"] + st["time_increment"] * (n - 1) == p["times"][1]
        assert st["imu_last"] == p["imu_last"], (name, j, st["imu_last"], p["imu_last"])
        if flags[0]:
            assert nc.same(got["imu"][j][:, :p["imu"].shape[1]], p["imu"]), f"{name}: scan {j}'s IMU table differs"
        assert nc.same(np.array([st["odom_start_time"], st["odom_end_time"]]), p["times"][2:])
        assert nc.same(got["poses"][j], p["poses"]), f"{name}: scan {j}'s odometry poses differ"
        assert nc.same(st["odom_incre"], p["incre"]), f"{name}: scan {j}'s odometry increment differs"


def test_streams_reach_their_cases():
    """Each named recording exercises what it is meant to."""
    def status(name):
        rec, flags, _ = nc.recording(name)
        return nc.restated(rec, flags)

    def has(name, *codes):
        s = list(status(name)["status"])
        return all(c in s for c in codes)

    assert has("late_imu", DS.WAIT_IMU, DS.PUBLISHED)
    g = status("imu_gap_start")
    assert g["status"][2] == DS.UNDEFINED and (g["status"][3:-1] == DS.PUBLISHED).all()
    g = status("imu_gap_whole")
    assert g["status"][2] == DS.PUBLISHED and g["state"]["imu_last"][2] == -1
    g = status("imu_over_2000")
    assert g["status"][2] == DS.UNDEFINED and g["state"]["imu_last"][2] == -2 and (g["status"][3:-1] == DS.PUBLISHED).all()
    assert has("imu_out_of_order", DS.WAIT_IMU, DS.PUBLISHED)
    g = status("odom_at_first_start")
    assert g["status"][0] == DS.PUBLISHED and g["state"]["odom_start_time"][0] == 0 and np.isnan(g["xyz"][0]).any()
    g = status("odom_sparse")
    pub = g["status"] == DS.PUBLISHED
    assert (g["state"]["odom_end_time"][pub] < g["state"]["time_start"][pub]).any()  # a stale end_odom_msg_
    assert (g["state"]["odom_end_time"][pub] == g["state"]["odom_start_time"][pub]).any()  # an interval of zero length
    assert has("odom_sparse", DS.WAIT_ODOM)
    p = status("odom_pitch90")["poses"]
    assert (np.abs(p[..., 4]) == np.pi / 2).any()
    assert has("negative_time_increment", DS.ODOM_EMPTY)
    for i in (0, 1):
        for o in (0, 1):
            assert has(f"mixed_flags{i}{o}", DS.PUBLISHED)
    assert list(status("one_scan")["status"]) == [DS.HELD]
    assert list(status("two_scans")["status"]) == [DS.PUBLISHED, DS.HELD]


def _call(use_imu=1, use_odom=1, n_beams=4, scans=None, ranges=True, imu=True, odom=True, n_imu=3, n_odom=2,
          status=True, xyz=True):
    L = DS._bind()
    sc = DS.node_scans([(1, 0), (1, 100_000_000)], 1e-4, 0.1, 30.0, [1, 3], [1, 2]) if scans is None else scans
    S = len(sc)
    r = np.ones((S, n_beams), np.float32)
    im = DS.imu_log(np.array([(1, 0), (1, 1), (1, 2)]), np.zeros((3, 3)))
    od = DS.odom_log(np.array([(1, 0), (1, 1)]), np.zeros((2, 3)), np.tile([0, 0, 0, 1.0], (2, 1)))
    st, out = np.zeros(S, np.int32), np.zeros((S, max(n_beams, 1), 3), np.float32)
    return L.b2s_lidar_undistortion_node(use_imu, use_odom, -1.0, 0.01, n_beams, S, sc.ctypes.data if S or scans is None else None,
                                         r.ctypes.data if ranges else None, n_imu, im.ctypes.data if imu else None,
                                         n_odom, od.ctypes.data if odom else None, st.ctypes.data if status else None,
                                         None, out.ctypes.data if xyz else None, 0, None)


def test_refusals_need_no_device(pkg):
    """NULL arrays, negative counts, no beams, arrival counts that decrease or exceed their log and a NULL log whose
    flag is on are refused before any device is touched; an empty recording needs none; otherwise no device is an
    error, never a CPU fallback."""
    BAD = 1
    assert _call(ranges=False) == BAD and _call(status=False) == BAD and _call(xyz=False) == BAD
    assert _call(n_beams=0) == BAD and _call(n_imu=-1) == BAD and _call(n_odom=-1) == BAD
    assert _call(imu=False) == BAD and _call(odom=False) == BAD
    assert _call(use_imu=0, imu=False) != BAD and _call(use_odom=0, odom=False) != BAD
    sc = DS.node_scans([(1, 0), (1, 1)], 1e-4, 0.1, 30.0, [2, 1], [1, 2])
    assert _call(scans=sc) == BAD  # IMU arrivals decrease
    sc = DS.node_scans([(1, 0), (1, 1)], 1e-4, 0.1, 30.0, [1, 4], [1, 2])
    assert _call(scans=sc) == BAD  # more IMU messages than the log holds
    sc = DS.node_scans([(1, 0), (1, 1)], 1e-4, 0.1, 30.0, [1, 3], [0, 3])
    assert _call(scans=sc) == BAD  # more odometry messages than the log holds
    sc = DS.node_scans([(1, 0)], 1e-4, 0.1, 30.0, [-1], [0])
    assert _call(scans=sc) == BAD
    L = DS._bind()
    assert L.b2s_lidar_undistortion_node(1, 1, 0.0, 0.01, 4, 0, C.c_void_p(8), C.c_void_p(8), 0, C.c_void_p(8), 0,
                                         C.c_void_p(8), C.c_void_p(8), None, C.c_void_p(8), 0, None) == 0
    assert L.b2s_lidar_undistortion_node(1, 1, 0.0, 0.01, 4, -1, C.c_void_p(8), C.c_void_p(8), 0, C.c_void_p(8), 0,
                                         C.c_void_p(8), C.c_void_p(8), None, C.c_void_p(8), 0, None) == BAD
    if pkg.load("matcher").device_count() == 0:
        assert _call() == 5  # B2S_ERR_NO_DEVICE
