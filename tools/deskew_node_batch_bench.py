"""Time lesson5's de-skew nodes behind one handle (b2s_deskew_node_*) against B one-shot calls: B seeded synthetic
recordings of 2000 scans of 1081 beams at 10 Hz with 200 Hz IMU and 50 Hz odometry, both flags on
(tests/deskew_node_cases.synthetic), for B in 1, 32 and 132.

  python tools/deskew_node_batch_bench.py [--batches 1,32,132] [--scans 2000] [--beams 1081]

Routes, each timed with the host clock around calls that end in a device synchronise:
  - whole: one handle call with every recording whole;
  - chunk100: the handle fed 100 scans of every recording per call;
  - per_scan: the handle fed one scan of every recording per call (a live robot's case), with the messages delivered
    since the previous scan;
  - one_shot: B b2s_lidar_undistortion_node calls in turn.
The handle's rows are callback-indexed (row k + 1 is the one-shot call's row k); every route must give the same
statuses and clouds bit for bit (NaN equal to NaN), else the script fails.  Prints one JSON line with the card's name
and power limit, read in the same run.  It needs a CUDA device; there is no CPU fallback.
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
DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def same(a, b):
    """bit equality, NaN equal to NaN at any payload"""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a).view(np.int32), np.where(nb, 0, b).view(np.int32))


def run_handle(recs, cut_every, want):
    """Feed every recording through one handle in calls of cut_every scans (0: whole) and compare every call's rows
    with `want` (per recording: status, xyz in the handle's row order) as they come.  -> seconds inside the calls."""
    S = len(recs[0]["scans"])
    cuts = list(range(cut_every, S, cut_every)) if cut_every else []
    plans = [DS.split_recording(r, cuts) for r in recs]
    h = DS.DeskewNodeBatch([DS.laser_of(r, (1, 1)) for r in recs])
    at, total = 0, 0.0
    for c in range(len(cuts) + 1):
        chunks = [p[c] for p in plans]
        t = time.perf_counter()
        got = h.process(chunks)
        total += time.perf_counter() - t
        k = len(chunks[0][0])
        for b, (status, _, xyz) in enumerate(got):
            if not (np.array_equal(status, want[b][0][at:at + k]) and same(xyz, want[b][1][at:at + k])):
                raise SystemExit(f"recording {b}: calls of {cut_every} scans differ from the one-shot calls at scan {at}")
        at += k
    h.close()
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,32,132")
    ap.add_argument("--scans", type=int, default=2000)
    ap.add_argument("--beams", type=int, default=1081)
    args = ap.parse_args()
    import deskew_node_cases as nc

    if DS.lib().b2s_device_count() < 1:
        raise SystemExit("no CUDA device: the de-skew nodes have no CPU fallback")
    gpu = card()
    warm = nc.synthetic(20, args.beams, seed=1)
    DS.undistort_recording(1, 1, warm["amin"], warm["ainc"], warm["scans"], warm["ranges"], warm["imu"], warm["odom"])
    DS.DeskewNodeBatch([DS.laser_of(warm, (1, 1))]).process([DS.split_recording(warm, [])[0]])
    results = []
    for B in (int(x) for x in args.batches.split(",")):
        recs = [nc.synthetic(args.scans, args.beams, seed=1000 + b) for b in range(B)]
        # B one-shot calls in turn; their rows, shifted to the handle's, are what every handle route must give
        want, t = [], time.perf_counter()
        for r in recs:
            status, _, xyz = DS.undistort_recording(1, 1, r["amin"], r["ainc"], r["scans"], r["ranges"], r["imu"], r["odom"])
            want.append((status, xyz))
        one_shot = time.perf_counter() - t
        want = [(np.concatenate([[DS.CACHED], s[:-1]]).astype(np.int32),
                 np.concatenate([np.zeros((1,) + x.shape[1:], np.float32), x[:-1]])) for s, x in want]
        row = {"recordings": B, "scans": B * args.scans, "beams": args.beams,
               "published": int(sum((w[0] == DS.PUBLISHED).sum() for w in want)), "one_shot_ms": one_shot * 1e3}
        for label, every in (("whole", 0), ("chunk100", 100), ("per_scan", 1)):
            row[label + "_ms"] = run_handle(recs, every, want) * 1e3
        for label in ("one_shot", "whole", "chunk100", "per_scan"):
            row[label + "_scans_per_s"] = row["scans"] / (row[label + "_ms"] * 1e-3)
        results.append(row)
        del recs, want
    print(json.dumps({"tool": "deskew_node_batch_bench", "card": gpu, "identical_clouds": True,
                      "imu_hz": 200, "odom_hz": 50, "results": results}))


if __name__ == "__main__":
    main()
