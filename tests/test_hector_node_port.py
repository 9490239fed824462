"""CPU tests of the lesson4 Hector SLAM node's restatement (oracle/hector_node_port.py): the publish schedule, the
squared-threshold arithmetic, the full-basis conversion against the yaw-only one where they must agree, and
InitParams over the shipped launch file."""
import math

import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P
from oracle import hector_scans_port as S

f32 = np.float32


def _run(period, stamps):
    s = P.Schedule(period)
    return [s.before(t) for t in stamps]


def test_schedule_first_scan_is_tick_zero():
    st = cases.stamps_at(100, 0, 25_000_000, 3)
    assert _run(2.0, st) == [(100, 0), None, None]


def test_schedule_tick_exactly_on_a_stamp_across_a_carry():
    # tick 0 = 10.9 s, tick 1 = 11.2 s = scan 2's stamp: published (>=), stamped 11.2 s
    assert _run(0.3, cases.exact_tick_stamps()) == [(10, 900_000_000), None, (11, 200_000_000), None]


def test_schedule_no_catch_up_over_gaps():
    st = cases.stamps_at(10, 900_000_000, 25_000_000, 6, gaps=((4, 5_000_000_000),))
    got = _run(0.3, st)
    # one publish after the gap, stamped with the earliest unpublished tick; the next tick is the first after 16.0 s
    assert got == [(10, 900_000_000), None, None, None, (11, 200_000_000), None]
    s = P.Schedule(0.3)
    for t in st[:5]:
        s.before(t)
    assert s.next == (16, 300_000_000)


def test_schedule_period_shorter_than_the_scan_interval():
    st = cases.stamps_at(1, 0, 25_000_000, 4)
    assert _run(0.01, st) == [(1, 0), (1, 10_000_000), (1, 30_000_000), (1, 60_000_000)]


def test_schedule_stamps_going_back_publish_nothing():
    st = np.array([(5, 0), (4, 0), (5, 100_000_000), (5, 0)], np.uint32)
    assert _run(0.1, st) == [(5, 0), None, (5, 100_000_000), None]


def test_duration_from_sec_rounds_half_away_from_zero():
    assert P.duration_from_sec(2.0) == (2, 0)
    assert P.duration_from_sec(0.3) == (0, 300_000_000)
    assert P.duration_from_sec(1.9999999999) == (2, 0)  # a whole second rolled over
    assert P.duration_from_sec(0.0000000005) == (0, 1)


@pytest.mark.parametrize("d", [0.2, 0.1, 0.05])
def test_squared_thresholds_round_the_double_square(d):
    node = P.sqr_threshold(d)
    assert node == f32(d * d)
    assert node != f32(d) * f32(d)  # the float square is one ulp above at these defaults


def test_beam_on_the_004f_boundary_is_kept_by_the_node():
    pts = np.array([[f32(0.2), 0.0, 0.0]], np.float32)
    kept, _ = P.to_data_container(pts, cases.mount(), 20.0, min_dist=0.2)
    assert len(kept) == 1
    yaw_only, _ = S.to_data_container(pts, (0, 0, 0, 0), 20.0, min_dist=0.2)
    assert len(yaw_only) == 0  # b2s_hector_scan_filter's float square drops it


def test_identity_and_translation_mounts_equal_the_yaw_only_conversion():
    rng = np.random.default_rng(3)
    pts = np.zeros((500, 3), np.float32)
    pts[:, :2] = rng.uniform(-25, 25, (500, 2)).astype(np.float32)
    for lb in [(0.0, 0.0, 0.0), (0.125, -0.0625, 0.25)]:
        a, oa = P.to_data_container(pts, cases.mount(*lb), 20.0, min_dist=0.25, max_dist=30.0)
        b, ob = S.to_data_container(pts, lb + (0.0,), 20.0, min_dist=0.25, max_dist=30.0)
        assert np.array_equal(a.view(np.int32), b.view(np.int32)) and np.array_equal(oa, ob)


def test_upside_down_mount_mirrors_y():
    pts = np.array([[1.0, 0.5, 0.0], [2.0, -1.5, 0.0]], np.float32)
    dc, _ = P.to_data_container(pts, cases.mount(0, 0, 0.3, roll=math.pi), 1.0)
    assert np.allclose(dc, [[1.0, -0.5], [2.0, 1.5]], atol=1e-6)


def test_pitched_mount_z_window_drops_far_beams():
    pts = np.array([[1.0, 0.0, 0.0], [10.0, 0.0, 0.0]], np.float32)
    dc, _ = P.to_data_container(pts, cases.mount(0, 0, 0.4, pitch=0.12), 1.0, z_min=-0.3, z_max=0.3)
    assert len(dc) == 1  # at 10 m the pitched beam is ~1.2 m below the laser


def test_shipped_launch_params():
    p = cases.hector_node.node_params(cases.hector_node.SHIPPED_LAUNCH)
    assert p.map_multi_res_levels == 3 and p.map_pub_period == 2.0 and p.map_update_angle_thresh == 0.9
    assert p.use_max_scan_range == 20.0 and p.laser_max_dist == 30.0 and p.map_size == 2048
    d = cases.hector_node.node_params()
    assert (d.map_resolution, d.laser_min_dist, d.laser_z_min_value, d.update_factor_occupied) == (0.05, 0.2, -1.0, 0.9)


def test_map_info_is_set_map_info_of_level_0():
    info = P.map_info(0.05, 2048, 0.5, 0.5)
    assert info["width"] == info["height"] == 2048 and info["resolution"] == float(f32(0.05))
    assert abs(info["origin_x"] + 51.2 + 0.025) < 1e-5 and info["origin_x"] == info["origin_y"]


def test_pose_message_fields():
    msg, cov, tf = P.pose_message(np.array([1.5, -2.0, 0.7], np.float32), np.arange(9, dtype=np.float32))
    half = float(f32(0.7) * f32(0.5))
    assert msg == [1.5, -2.0, 0.0, 0.0, 0.0, math.sin(half), math.cos(half)]
    nz = {0: 0, 7: 4, 35: 8, 1: 1, 6: 1, 5: 2, 30: 2, 11: 5, 31: 5}
    assert all(cov[k] == (nz[k] if k in nz else 0) for k in range(36))
    assert np.allclose(tf, msg, atol=1e-15)


def test_port_runs_a_recording_with_publishes():
    c = cases.cases()["short_period"]
    node = P.HectorNodePort(c["params"], c["geometry"], c["mount"])
    out = node.process(c["ranges"][:3], c["stamps"][:3])
    node.close()
    assert [m["scan_index"] for m in out["maps"]] == [0, 1, 2]
    assert (out["maps"][0]["payload"] == -1).all() and out["maps"][0]["rebuilt"]
    assert out["maps"][1]["rebuilt"] and (out["maps"][1]["payload"] != -1).any()
