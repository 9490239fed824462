"""lesson5 motion de-skew against the unmodified node and an independent float64 reference (CPU).

The node (reference/lesson5/src/lidar_undistortion.cc) is compiled where it lies against ROS, tf, PCL and Eigen stand-ins
(oracle/ref_lesson5.cpp) and fed whole message streams through its callbacks, live where oracle/_ref/ is built and from
tests/golden/reference/ elsewhere.  Every line of the node that runs is pinned; pcl::getTransformation, Eigen's Affine3f
inverse and product and tf's getRPY are stand-ins that restate the same algorithms as the kernel, so they are not.
tests/deskew_reference.py checks the geometry itself in float64 within a bound derived from float32 rounding."""
import numpy as np
import pytest

import deskew_cases as dc
import deskew_reference as dr
from oracle import port, ref_lesson5


@pytest.fixture(scope="module")
def answers():
    return dc.node_answers(ref_lesson5.available())


@pytest.mark.parametrize("name", sorted(dc.NODE_STREAMS))
def test_restatement_equals_node(pkg, answers, name):
    """The C restatement, fed the library's IMU table and odometry increment (which must equal the node's own), returns
    the node's published cloud bit for bit; the float64 reference agrees with both within its bound."""
    st, pubs, flags = answers[name]
    got = []
    for pub in pubs:
        k, ranges, amin, ainc, info, tab = dc.abi_inputs(pkg, st, pub, flags)
        got.append(k)
        want = port.deskew_scan(ranges, amin, ainc, info, *tab)
        diff = want.view(np.int32) != pub["xyz"].view(np.int32)
        assert not diff.any(), f"scan {k}: {diff.any(1).sum()} beams differ from the node, first {np.argwhere(diff)[0]}"
        dr.check(pub["xyz"], ranges, amin, ainc, info, *tab)
    assert got == dc.NODE_PUBLISHED.get(name, list(range(len(st["scans"]) - 1)))


def test_node_streams_reach_the_edges(pkg, answers):
    """The streams cover what they are meant to: roll and pitch above 1.3 rad, yaw past pi, imu_last 0, first valid
    beams at 0, 255, 256, 700 and n - 1, a scan without a valid beam, and every kept / dropped range edge."""
    st, pubs, _ = answers["slabs"]
    assert max(np.abs(p["imu"][1]).max() for p in pubs) > 1.3 and max(np.abs(p["imu"][2]).max() for p in pubs) > 1.3
    assert max(np.abs(p["imu"][3]).max() for p in pubs) > np.pi
    assert all(p["imu_last"] == 0 for p in answers["imu_last0"][1])
    for k, fv in enumerate((0, 255, 256, 700, 1080)):
        assert np.argmax(dr.valid(st["scans"][k][3], dict(range_min=0.1, range_max=30.0))) == fv
    st, pubs, _ = answers["validity"]
    assert list(dr.valid(st["scans"][0][3][:12], dict(range_min=0.25, range_max=20.0))) == \
        [True, True, False, False, False, False, False, False, False, False, False, True]
    assert list(dr.valid(st["scans"][1][3][:8], dict(range_min=0.0, range_max=20.0))) == \
        [True, True, True, False, False, True, False, True]
    assert not pubs[2]["xyz"].any()


def test_beam_angles_are_summed_in_float32():
    """CreateAngleCache sums float fields: at the 1081-beam geometry most angles differ from the double sum."""
    n = 1081
    a32 = dr.beam_angles(n, np.float32(-2.35619449), np.float32(4.71238898 / 1080))
    a64 = float(np.float32(-2.35619449)) + np.arange(n) * float(np.float32(4.71238898 / 1080))
    assert (a32 != a64).sum() > 1000 and np.abs(a32 - a64).max() < 3e-7


@pytest.mark.parametrize("case", sorted(dc.ABI_CASES))
def test_restatement_within_the_float64_bound(pkg, case):
    """Inputs only the ABI can express (hand-made IMU tables, odometry intervals inside the scan, negative time
    increments, sentinels past imu_last): the restatement within the float64 reference's bound."""
    for ranges, amin, ainc, info, tab in dc.ABI_CASES[case](pkg):
        dr.check(port.deskew_scan(ranges, amin, ainc, info, *tab), ranges, amin, ainc, info, *tab)
