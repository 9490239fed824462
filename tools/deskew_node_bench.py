"""Time lesson5's whole de-skew node on a recording: b2s_lidar_undistortion_node over a seeded synthetic recording of
10 000 scans of 1081 beams at 10 Hz with 200 Hz IMU and 50 Hz odometry, both flags on, host arrays in and clouds out
(tests/deskew_node_cases.synthetic).

  python tools/deskew_node_bench.py [--scans 10000] [--beams 1081] [--warmup 2] [--repeats 7]

Prints one JSON line:
  - node_ms / scans_per_s: the call, with a device synchronise, inside the timed region (median, min, max of the
    repeats); h2d_bytes / d2h_bytes: what the call copies each way;
  - batch_ms: the route without the node call: the node's queues, IMU integration and odometry increments prepared
    per scan on the host (b2s_deskew_integrate_imu, tf's getRPY restated in Python, b2s_deskew_odom_increment), then
    one b2s_lidar_undistort batch (median of the repeats);
  - cpu_ms: the C restatement (oracle/deskew_node_oracle.c) on one core, once;
  - the card's name and power limit, read in the same run.
All three routes must give the same clouds (NaN equal to NaN).  It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def get_rpy(q):
    """tf::quaternionMsgToTF + Matrix3x3(q).getRPY, in Python floats (the C library's atan2 / asin / cos)"""
    x, y, z, w = (float(v) for v in q)
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d if d != 0 else math.nan
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz, xx, xy, xz, yy, yz, zz = w * xs, w * ys, w * zs, x * xs, x * ys, x * zs, y * ys, y * zs, z * zs
    m00, m01, m02, m10 = 1.0 - (yy + zz), xy - wz, xz + wy, xy + wz
    m20, m21, m22 = xz - wy, yz + wx, 1.0 - (xx + yy)
    if abs(m20) >= 1:
        return (math.atan2(-m01, -m02), -math.pi / 2, 0.0) if m20 > 0 else (0.0 + math.atan2(m01, m02), math.pi / 2, 0.0)
    pitch = -math.asin(m20)
    c = math.cos(pitch)
    return math.atan2(m21 / c, m22 / c), pitch, math.atan2(m10 / c, m00 / c)


def batch_route(rec):
    """the node's callbacks prepared per scan on the host, then one b2s_lidar_undistort call -> clouds [S, n, 3]"""
    sc, r = rec["scans"], rec["ranges"]
    S, n = r.shape
    it = rec["imu"]["sec"].astype(np.float64) + 1e-9 * rec["imu"]["nsec"].astype(np.float64)
    ot = rec["odom"]["sec"].astype(np.float64) + 1e-9 * rec["odom"]["nsec"].astype(np.float64)
    starts = sc["sec"].astype(np.float64) + 1e-9 * sc["nsec"].astype(np.float64)
    ilo = olo = 0
    sm = em = -1
    rows, infos, tabs = [], [], []
    for j in range(S - 1):
        start, inc = float(starts[j]), float(sc["time_increment"][j])
        end = start + inc * (float(n) - 1)
        ihi, ohi = int(sc["imu_arrived"][j + 1]), int(sc["odom_arrived"][j + 1])
        if ilo == ihi or it[ilo] > start or it[ihi - 1] < end:
            continue
        while ilo < ihi and it[ilo] < start - 0.1:
            ilo += 1
        if ilo == ihi:
            continue
        last, *tab = DS.integrate_imu(it[ilo:ihi], rec["imu"]["angular_velocity"][ilo:ihi], start, end)
        if olo == ohi or ot[olo] > start or ot[ohi - 1] < end:
            continue
        while olo < ohi and ot[olo] < start - 0.1:
            olo += 1
        if olo == ohi:
            continue
        for i in range(olo, ohi):
            if ot[i] < start:
                sm = i
            elif ot[i] <= end:
                em = i
            else:
                break
        assert last >= 0 and sm >= 0 and em >= 0, "the benchmark recording has no undefined or default-message scans"
        poses = [np.concatenate([rec["odom"]["position"][m], get_rpy(rec["odom"]["orientation"][m])]) for m in (sm, em)]
        info = DS.DeskewScan()
        info.time_start, info.time_increment = start, inc
        info.range_min, info.range_max = sc["range_min"][j], sc["range_max"][j]
        info.use_imu = info.use_odom = 1
        info.imu_last, info.odom_start_time, info.odom_end_time = last, ot[sm], ot[em]
        info.odom_incre[:] = DS.odom_increment(*poses)
        rows.append(j)
        infos.append(info)
        tabs.append([t[:last + 1] for t in tab])
    stride = max(len(t[0]) for t in tabs)
    T = [np.stack([np.pad(t[a], (0, stride - len(t[a]))) for t in tabs]) for a in range(4)]
    out = np.zeros((S, n, 3), np.float32)
    out[rows] = DS.undistort(r[rows], rec["amin"], rec["ainc"], infos, *T)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=10_000)
    ap.add_argument("--beams", type=int, default=1081)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    import torch
    import deskew_node_cases as nc
    from oracle import deskew_node_port

    assert pkg_device_count() > 0, "no CUDA device: there is no CPU fallback"
    rec = nc.synthetic(a.scans, a.beams, imu_hz=200, odom_hz=50, seed=2024)
    args = (1, 1, rec["amin"], rec["ainc"], rec["scans"], rec["ranges"], rec["imu"], rec["odom"])
    out = np.zeros((a.scans, a.beams, 3), np.float32)
    for _ in range(a.warmup):
        DS.undistort_recording(*args, out=out)
    times = []
    for _ in range(a.repeats):
        t = time.perf_counter()
        status, state, _ = DS.undistort_recording(*args, out=out)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    n_pub = int((status == DS.PUBLISHED).sum())
    batch_times = []
    for _ in range(max(1, a.repeats // 2)):
        t = time.perf_counter()
        via_batch = batch_route(rec)
        torch.cuda.synchronize()
        batch_times.append((time.perf_counter() - t) * 1e3)
    t = time.perf_counter()
    cpu = deskew_node_port.node(*args[:6], rec["imu"], rec["odom"])
    cpu_ms = (time.perf_counter() - t) * 1e3
    assert nc.same(out, cpu["xyz"]) and nc.same(out, via_batch), "the three routes give different clouds"
    n_imu = len(rec["imu"])
    h2d = rec["ranges"].nbytes + 8 * (2 * a.beams + 4 * n_imu) + n_pub * (DS.STATE_DTYPE.itemsize + 24)
    med = statistics.median(times)
    print(json.dumps(dict(
        workload=f"{a.scans} scans x {a.beams} beams, 200 Hz IMU, 50 Hz odometry, use_imu and use_odometry",
        published=n_pub, node_ms=dict(median=med, min=min(times), max=max(times)), scans_per_s=a.scans / med * 1e3,
        h2d_bytes=h2d, d2h_bytes=out.nbytes, batch_ms=statistics.median(batch_times),
        batch_scans_per_s=a.scans / statistics.median(batch_times) * 1e3, cpu_ms=cpu_ms,
        cpu_scans_per_s=a.scans / cpu_ms * 1e3, identical_clouds=True, card=card())))


def pkg_device_count():
    return importlib.import_module("creating-2d-laser-slam-from-scratch_b200.matcher").device_count()


if __name__ == "__main__":
    main()
