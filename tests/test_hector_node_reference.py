"""lesson4's Hector SLAM node (hector_slam.cc) restated in oracle/hector_node_port.py against the unmodified node (CPU).

The node is compiled where it lies against ROS, tf, laser_geometry and Boost stand-ins (oracle/ref_lesson4_slam.cpp),
live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere; maps are compared through digests.  Both
sides publish on the library's schedule (the node's own runs on a thread).  Pinned bit for bit: getLastScanMatchPose,
the odom_hector pose and covariance, both transforms sent (map -> odom stays the identity), the kept-beam count, and
every published map's payload, info and rebuild gate.  Rows before the first matched scan are left out of the
covariance: the node reads an uninitialised matrix there."""
import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P
from oracle import ref_lesson4_slam
from reference_record import digest, recording

CASES = cases.cases()
IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1.0])


def _params(c):
    p = cases.hector_node.node_params(c["params"])
    return {f: getattr(p, f) for f, _ in cases.hector_node.HectorNodeParams._fields_}


def _node(c):
    prm = _params(c)
    out = ref_lesson4_slam.run(prm, c["geometry"], c["mount"], c["ranges"], c["stamps"], P.Schedule(prm["map_pub_period"]))
    bad = cases.uninitialised_rows(out["n_points"])
    out["cov"][bad] = 0.0  # uninitialised memory in the node: not an answer
    out["maps"] = [dict(m, payload=digest(m["payload"])) for m in out["maps"]]
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_port_equals_node(request, name):
    c = CASES[name]
    live = ref_lesson4_slam.available()
    with recording(request, live) as rec:
        want = rec.value("node", lambda: _node(c), inputs=(name, _params(c), c["geometry"], c["mount"], c["ranges"],
                                                                   c["stamps"]))
    port = P.HectorNodePort(_params(c), c["geometry"], c["mount"])
    got = port.process(c["ranges"], c["stamps"])
    port.close()
    same = lambda a, b: np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    assert same(got["pose"], np.asarray(want["pose"], np.float32)), name
    assert np.array_equal(got["n_points"], want["n_points"]), name
    assert same(got["pose_msg"], np.asarray(want["pose_msg"], np.float64)), name
    keep = ~cases.uninitialised_rows(got["n_points"])
    assert same(got["cov"][keep], np.asarray(want["cov"], np.float64)[keep]), name
    tf = np.asarray(want["tf"], np.float64)
    assert all(same(t, IDENTITY) for t in tf[:, 0]), name  # map -> odom
    assert same(got["tf"], tf[:, 1]), name                 # odom -> base_link, poseMsgToTF of the pose
    assert len(got["maps"]) == len(want["maps"]), name
    for g, w in zip(got["maps"], want["maps"]):
        assert (g["scan_index"], tuple(g["stamp"]), g["rebuilt"]) == (int(w["scan_index"]), tuple(w["stamp"]), bool(w["rebuilt"]))
        for f in ("origin_x", "origin_y", "resolution", "width", "height"):
            assert g["info"][f] == w["info"][f], (name, f)
        assert digest(g["payload"]) == w["payload"], name


def test_cases_cover_the_node():
    c = CASES
    assert c["shipped_launch"]["mount"] == cases.mount(0, 0, 0.254, roll=3.1415926)  # the launch file's roll
    assert (c["boundary_0.04f"]["ranges"][:, 0] == np.float32(0.2)).all()
