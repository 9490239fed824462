"""Recordings for lesson6's Karto SLAM node (tests/test_karto_node_reference.py, tests/test_gpu_karto_node.py,
tools/karto_node_bench.py): a robot circling a room lap after lap (synth.make_loop_trajectory), ROS-shaped.  Each case
is a LaserScan geometry, float32 ranges, 10 Hz (sec, nsec) stamps, odom <- base_link rows (translation + quaternion;
NaN where the tf lookup fails), the laser mount and the node's ROS parameters."""
from __future__ import annotations

import importlib
import math
import os
import sys
from dataclasses import dataclass, field

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")

N_BEAMS = 1081
ANGLE_MIN = np.float32(math.radians(-135.0))
ANGLE_INC = np.float32(math.radians(0.25))

# small matcher windows (as tests/mapper_cases.py) keep the CPU reference fast; loops close on the second lap
SMALL = dict(use_scan_range=9.25, scan_buffer_size=20, link_match_minimum_response_fine=0.1, link_scan_maximum_distance=1.5,
             loop_search_maximum_distance=3.0, loop_match_minimum_chain_size=5, loop_match_maximum_variance_coarse=3.0,
             loop_match_minimum_response_coarse=0.35, loop_match_minimum_response_fine=0.45,
             correlation_search_space_dimension=0.5, correlation_search_space_resolution=0.05,
             loop_search_space_dimension=4.0)

# lesson6/config/mapper_params.yaml as shipped (its minimum_time_interval is never read by the node)
SHIPPED_YAML = dict(use_scan_matching=True, use_scan_barycenter=True, minimum_time_interval=3600,
                    minimum_travel_distance=0.2, minimum_travel_heading=0.174, scan_buffer_size=110,
                    scan_buffer_maximum_scan_distance=100.0, use_scan_range=12, correlation_search_space_dimension=0.3,
                    correlation_search_space_resolution=0.01, correlation_search_space_smear_deviation=0.03,
                    distance_variance_penalty=0.5, angle_variance_penalty=0.1, fine_search_angle_offset=0.00349,
                    coarse_search_angle_offset=0.349, coarse_angle_resolution=0.0349, minimum_angle_penalty=0.9,
                    minimum_distance_penalty=0.5, use_response_expansion=True, use_back_end=False, marker_count=0,
                    solver_type="spa_solver", loop_search_space_dimension=10.0, loop_search_space_resolution=0.05,
                    loop_search_space_smear_deviation=0.03, link_match_minimum_response_fine=0.1,
                    link_scan_maximum_distance=1.5, loop_search_maximum_distance=10.0, do_loop_closing=True,
                    loop_match_minimum_chain_size=5, loop_match_maximum_variance_coarse=3,
                    loop_match_minimum_response_coarse=0.35, loop_match_minimum_response_fine=0.45)


def quat_rpy(roll, pitch, yaw):
    """tf's Quaternion::setRPY"""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


@dataclass
class Case:
    name: str
    params: dict
    ranges: np.ndarray   # [S][n] float32
    stamps: np.ndarray   # [S][2] uint32
    odom: np.ndarray     # [S][7]
    mount: tuple = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    standard_geometry: bool = False  # angle_max = angle_min + (n - 1) * inc: the laser has n - 1 readings
    expect: set = field(default_factory=set)

    @property
    def fields(self):
        """(angle_min, angle_max, angle_increment, range_min, range_max) float32 as the message carries them"""
        n = self.ranges.shape[1]
        amax = ANGLE_MIN + np.float32(n - 1 if self.standard_geometry else n) * ANGLE_INC
        return np.array([ANGLE_MIN, amax, ANGLE_INC, 0.1, 30.0], np.float32)

    def geometry(self):
        f = self.fields
        return pkg.load("rosio").make_msg(f[0], f[1], f[2], f[3], f[4], np.zeros(self.ranges.shape[1], np.float32))

    @property
    def use_back_end(self):
        return bool(self.params.get("use_back_end", False))


def stamps_10hz(S, sec0=1000, nsec0=0):
    t = sec0 * 1_000_000_000 + nsec0 + np.arange(S, dtype=np.int64) * 100_000_000
    return np.stack([t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)


def odom_rows(poses):
    return np.array([(x, y, 0.0, 0.0, 0.0, math.sin(h * 0.5), math.cos(h * 0.5)) for x, y, h in poses], np.float64)


def recording(seed, S, n=N_BEAMS):
    laser = pkg.synth.Laser(type=0, n_readings=n, min_angle=float(ANGLE_MIN), max_angle=float(ANGLE_MIN + n * ANGLE_INC),
                            angular_resolution=float(ANGLE_INC), range_threshold=9.25)
    _, _, odom, ranges = pkg.synth.make_loop_trajectory(seed, S, laser, radius=2.0, step=0.25)
    return ranges.astype(np.float32), odom


def cases():
    out = []
    r, o = recording(1, 60)
    out.append(Case("defaults", {}, r, stamps_10hz(60), odom_rows(o), expect={"maps>=2"}))
    r, o = recording(2, 70)
    # its 110-scan running window keeps every scan of a short recording out of loop closing: near chains link instead
    out.append(Case("shipped_yaml", dict(SHIPPED_YAML), r, stamps_10hz(70), odom_rows(o), expect={"near_links", "maps>=2"}))
    r, o = recording(4, 80)
    out.append(Case("loops_small_windows", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(80), odom_rows(o),
                    expect={"loops", "maps>=2"}))
    r, o = recording(3, 45)
    out.append(Case("throttle_3", dict(SMALL, throttle_scans=3, map_update_interval=0.5), r, stamps_10hz(45), odom_rows(o),
                    expect={"throttled", "maps>=2"}))
    r, o = recording(4, 30)
    out.append(Case("interval_0", dict(SMALL, map_update_interval=0.0), r, stamps_10hz(30), odom_rows(o),
                    expect={"map_every_processed"}))
    out.append(Case("interval_1e6", dict(SMALL, map_update_interval=1e6), r, stamps_10hz(30), odom_rows(o),
                    expect={"one_map"}))
    r, o = recording(5, 30)
    out.append(Case("interval_exact", dict(SMALL, map_update_interval=0.3), r, stamps_10hz(30, 1000, 850_000_000),
                    odom_rows(o), expect={"exact_interval_no_map", "maps>=2"}))
    r, o = recording(7, 40)
    out.append(Case("mount_offset_yaw", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40), odom_rows(o),
                    mount=(0.2, -0.1, 0.3) + quat_rpy(0.0, 0.0, 0.3), expect={"maps>=2"}))
    out.append(Case("mount_upside_down", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40), odom_rows(o),
                    mount=(0.05, 0.0, 0.2) + quat_rpy(math.pi, 0.0, 0.0), expect={"inverted", "maps>=2"}))
    r, o = recording(5, 30)
    idx = [0, 1, 1, 1, 2, 3, 3, 4, 5, 6, 6, 6, 6, 7, 8, 9, 10, 10, 11, 12]  # the robot stands still now and then
    out.append(Case("standing_still", dict(SMALL, map_update_interval=0.5), r[idx], stamps_10hz(len(idx)),
                    odom_rows(o[idx]), expect={"not_moved", "maps>=2"}))
    r, o = recording(8, 40)
    od = odom_rows(o)
    od[[3, 4, 17, 30]] = np.nan
    od[22, 5] = np.nan
    out.append(Case("odom_failures", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40), od,
                    expect={"no_odom", "maps>=2"}))
    r, o = recording(7, 40)
    rng = np.random.default_rng(8)
    for i in range(40):
        k = rng.choice(N_BEAMS, 40, replace=False)
        r[i, k[:10]] = np.nan
        r[i, k[10:20]] = np.inf
        r[i, k[20:30]] = 0.05   # below range_min
        r[i, k[30:]] = 45.0     # beyond range_max
    out.append(Case("bad_readings", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40), odom_rows(o),
                    expect={"maps>=2"}))
    r, o = recording(2, 40)
    out.append(Case("standard_geometry", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40), odom_rows(o),
                    standard_geometry=True, expect={"last_beam_dropped", "maps>=2"}))
    out.append(Case("standard_geometry_upside_down", dict(SMALL, map_update_interval=1.0), r, stamps_10hz(40),
                    odom_rows(o), mount=(0.0, 0.0, 0.1) + quat_rpy(math.pi, 0.0, 0.0), standard_geometry=True,
                    expect={"last_beam_dropped", "inverted", "maps>=2"}))
    r, o = recording(3, 80)
    out.append(Case("back_end", dict(SMALL, use_back_end=True, map_update_interval=1.0), r, stamps_10hz(80),
                    odom_rows(o), expect={"loops", "poses_moved", "maps>=2"}))
    return out


def pose_graph():
    """A fresh back end for one node (use_back_end): the library's pose-graph optimiser as a ScanSolver"""
    return pkg.load("mapper").PoseGraph().as_scan_solver()


CASES = {c.name: c for c in cases()}
