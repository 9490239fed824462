"""Time lesson4's Hector SLAM node handle (b2s_hector_node_process) on a whole recording: a seeded synthetic walk of
1081-beam scans (Hokuyo UTM-30LX geometry) at 40 Hz, the node's default parameters (2048 x 2048 level 0, three levels)
with map_pub_period 2 s, host ranges in and every published map handed to a callback on the host.

  python tools/hector_node_bench.py [--scans 10000] [--repeats 3]

Prints one JSON line:
  - scans_per_s / ms: the handle over the whole recording (median of the repeats; maps counted, not kept);
  - publish_share: 1 - (the same recording with map_pub_period 1e6 s, one publish) / (the run at 2 s);
  - route_parts_*: the same work through the existing calls, batched: b2s_hector_slam_process_scans_batch over the
    parts between publish points plus b2s_hector_slam_copy_level_ros at each;
  - route_per_scan_*: the existing calls one scan at a time, as a caller without the handle drives them: one
    b2s_hector_slam_process_scans_batch call per scan plus b2s_hector_slam_copy_level_ros at each publish point, over the
    first --per-scan scans.
  The existing calls take the mount as x, y, z, yaw (the identity here) and square the range thresholds in float, so a
  beam on the 0.04f boundary would go the other way; the recording has none.
  - kernel: the stream kernel the handle launches, and the card's name and power limit, read in the same run.
It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def recording(n, laser):
    """n scans: a 500-scan walk repeated forwards and backwards (no jumps), 40 Hz stamps."""
    synth = pkg.synth
    _, _, base = synth.make_trajectory(5, 500, laser, step_xy=0.02, step_th_deg=0.5)
    base = base.astype(np.float32)
    loop = np.concatenate([base, base[::-1]])
    r = np.ascontiguousarray(np.resize(loop, (n, laser.n_readings)), np.float32)
    t = 1_000 * 1_000_000_000 + np.arange(n, dtype=np.int64) * 25_000_000
    return r, np.stack([t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)


def run_node(N, geom, r, st, period):
    node = N.HectorNode(N.node_params(dict(map_pub_period=period)), geom)
    count = [0]
    t0 = time.perf_counter()
    out = node.process(r, st, on_map=lambda m: count.__setitem__(0, count[0] + 1))
    ms = (time.perf_counter() - t0) * 1e3
    node.close()
    return ms, count[0], out


def run_route(H, R, geom, r, cuts):
    """process_scans_batch between publish points, copy_level_ros at each."""
    h = H.HectorSlam(resolution=0.05, size_x=2048, size_y=2048, levels=3, min_dist=0.4, min_angle=0.9, batch=1,
                     max_points=r.shape[1])
    filt = R.hector_scan_filter()
    edges = list(cuts) + [len(r)]
    t0 = time.perf_counter()
    first = np.zeros((1, 3), np.float32)
    for a, b in zip(edges[:-1], edges[1:]):
        h.ros_map_of(0, 0)
        if b > a:
            res, _, _ = h.process_scans_batch(geom, [r[a:b]], filt, first_hints=first)
            first = res[0][0][-1:].copy()
    ms = (time.perf_counter() - t0) * 1e3
    h.close()
    return ms


def run_per_scan(H, R, geom, r, cuts):
    """One process_scans_batch call per scan, copy_level_ros at each publish point."""
    h = H.HectorSlam(resolution=0.05, size_x=2048, size_y=2048, levels=3, min_dist=0.4, min_angle=0.9, batch=1,
                     max_points=r.shape[1])
    filt = R.hector_scan_filter()
    due = set(cuts)
    t0 = time.perf_counter()
    for i in range(len(r)):
        if i in due:
            h.ros_map_of(0, 0)
        h.process_scans_batch(geom, [r[i:i + 1]], filt)
    ms = (time.perf_counter() - t0) * 1e3
    h.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--per-scan", type=int, default=2000)
    a = ap.parse_args()
    M = pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("hector_node_bench: no CUDA device (there is no CPU fallback)")
    N, H, R = pkg.load("hector_node"), pkg.load("hector"), pkg.load("rosio")
    laser = pkg.synth.Laser()
    r, st = recording(a.scans, laser)
    amin, inc = np.float32(laser.min_angle), np.float32(laser.angular_resolution)
    geom = R.make_msg(amin, amin + inc * np.float32(laser.n_readings - 1), inc, np.float32(0.1), np.float32(30.0),
                      np.zeros(laser.n_readings, np.float32))
    run_node(N, geom, r[:200], st[:200], 2.0)  # warm-up: module load, pools, page-locked buffers
    runs = [run_node(N, geom, r, st, 2.0) for _ in range(a.repeats)]
    ms = statistics.median(x[0] for x in runs)
    n_maps = runs[0][1]
    quiet = statistics.median(run_node(N, geom, r, st, 1e6)[0] for _ in range(a.repeats))
    # the publish points of the 2 s schedule (every 80th scan at 40 Hz)
    cuts = [0] + [i for i in range(1, len(st)) if (st[i, 0] - st[0, 0]) // 2 != (st[i - 1, 0] - st[0, 0]) // 2]
    route = statistics.median(run_route(H, R, geom, r, cuts) for _ in range(a.repeats))
    k = min(a.per_scan, a.scans)
    per_scan = statistics.median(run_per_scan(H, R, geom, r[:k], [c for c in cuts if c < k]) for _ in range(a.repeats))
    print(json.dumps(dict(
        scans=a.scans, beams=laser.n_readings, maps=n_maps, ms=round(ms, 1), scans_per_s=round(a.scans / ms * 1e3),
        publish_share=round(1.0 - quiet / ms, 3), ms_one_publish=round(quiet, 1),
        route_parts_ms=round(route, 1), route_parts_scans_per_s=round(a.scans / route * 1e3), route_maps=len(cuts),
        route_per_scan_scans=k, route_per_scan_ms=round(per_scan, 1), route_per_scan_scans_per_s=round(k / per_scan * 1e3),
        kernel="k_hs_stream_batch<true, true> (one CTA, exact mode)", card=card())))


if __name__ == "__main__":
    main()
