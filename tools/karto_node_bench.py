"""Time lesson6's Karto SLAM node on a long recording: b2s_karto_node_process over a seeded synthetic recording (a robot
circling a 9 m radius lap after lap in a 28 m x 24 m hall with 12 boxes, synth.make_loop_trajectory, 1081 beams, 10 Hz)
at the shipped config/mapper_params.yaml values (tests/karto_node_cases.SHIPPED_YAML), with the node's default 5 s map
interval.

  python tools/karto_node_bench.py [--scans 3000] [--step 0.25]

Prints one JSON line:
  - node_s, scans_per_s, key_frames_per_s: the whole recording in one call, end to end (host arrays in, every map
    handed out);
  - map_updates, map_s and map_share: how many maps were built, and the time the per-scan route below spends building
    the same maps (b2s_occ_grid_create_from_scans + copy_ros, the calls the node makes), as a share of node_s;
  - per_scan_s: the same recording through the per-scan route from Python (b2s_mapper_process_sensor per scan, the
    tf arithmetic restated in Python, b2s_occ_grid_create_from_scans + copy_ros whenever the node publishes), whose
    poses and maps must equal the node's;
  - the card's name and power limit, read in the same run.
It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
KN = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.karto_node")
MP = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.mapper")
OG = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.occgrid")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def per_scan_route(c, got):
    from oracle import karto_node_port as P
    prm, _ = KN.node_params(c.params)
    laser, inverted = P.laser_of(c.geometry(), c.mount, prm.use_scan_range)
    prm.mapper.sequential.range_threshold = prm.mapper.loop.range_threshold = laser.range_threshold
    m = MP.Mapper(prm.mapper, laser)
    ident = (P._rotation(P._quat_rpy(0.0, 0.0, 0.0)), [0.0, 0.0, 0.0])
    kept, maps, last, map_s = [], [], None, 0.0
    t0 = time.perf_counter()
    for i in range(len(c.ranges)):
        op = P._mul(P._from_row(c.odom[i]), ident)
        r = c.ranges[i][:laser.n_readings].astype(np.float64)
        ok, pose = m.process(r, (op[1][0], op[1][1], P._yaw(P._quaternion(op[0]))), 0.0, sensor="laser")
        if not ok:
            continue
        kept.append(r)
        s = (int(c.stamps[i][0]), int(c.stamps[i][1]))
        if last is None or P.stamp_diff(s, last) > P.duration_from_sec(prm.map_update_interval):
            t1 = time.perf_counter()
            g = OG.OccupancyGrid(laser, np.array(kept), m.poses(), prm.resolution)
            maps.append((i, g.ros_map()))
            g.close()
            map_s += time.perf_counter() - t1
            last = s
    dt = time.perf_counter() - t0
    assert [i for i, _ in maps] == [i for i, _, _ in got["maps"]], "the per-scan route publishes different maps"
    assert all(np.array_equal(a, b[2]) for (_, a), b in zip(maps, got["maps"])), "the per-scan route's maps differ"
    assert np.array_equal(m.poses(), got["poses"]), "the per-scan route's poses differ"
    m.close()
    return dt, map_s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=3000)
    ap.add_argument("--step", type=float, default=0.25)
    a = ap.parse_args()
    import karto_node_cases as kc
    laser = kc.pkg.synth.Laser(type=0, n_readings=kc.N_BEAMS, min_angle=float(kc.ANGLE_MIN),
                               max_angle=float(kc.ANGLE_MIN + kc.N_BEAMS * kc.ANGLE_INC),
                               angular_resolution=float(kc.ANGLE_INC), range_threshold=12.0)
    _, _, odom, ranges = kc.pkg.synth.make_loop_trajectory(11, a.scans, laser, radius=9.0, step=a.step, half_w=14.0,
                                                           half_h=12.0, n_boxes=12)
    c = kc.Case("bench", dict(kc.SHIPPED_YAML), ranges.astype(np.float32), kc.stamps_10hz(a.scans), kc.odom_rows(odom))
    prm, _ = KN.node_params(c.params)

    def run(interval):
        prm.map_update_interval = interval
        node = KN.KartoNode(prm, c.geometry(), c.mount)
        t0 = time.perf_counter()
        out = node.process(c.ranges, c.stamps, c.odom)
        dt = time.perf_counter() - t0
        out["poses"] = node.mapper.poses()
        out["stats"] = node.mapper.stats()
        node.close()
        return dt, out

    run(5.0)  # warm-up: the CUDA context and the kernels' first launches
    node_s, got = run(5.0)
    per_scan_s, map_s = per_scan_route(c, got)
    key = int((got["state"] == KN.PROCESSED).sum())
    print(json.dumps(dict(scans=a.scans, beams=kc.N_BEAMS, key_frames=key, node_s=round(node_s, 3),
                          scans_per_s=round(a.scans / node_s, 1), key_frames_per_s=round(key / node_s, 1),
                          map_updates=len(got["maps"]), map_s=round(map_s, 3), map_share=round(map_s / node_s, 3),
                          loops_closed=got["stats"]["loops_closed"], per_scan_s=round(per_scan_s, 3), card=card())))


if __name__ == "__main__":
    main()
