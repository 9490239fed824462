"""Throughput and latency of the lesson3 PL-ICP odometry node on the device (b2s_plicp_odom_process).

  python tools/plicp_odometry_bench.py [--fleets 132,1024] [--scans 100] [--latency-scans 200]

Recordings are synthetic drives (synth.py, 1081 beams) built from a pool of scans along one trajectory; recording b
starts at pool offset b.  Reports, with the card's name and power limit read in the same run:
  * scans/s end to end (host ranges in, outputs on the host) for B recordings x S scans in one call;
  * per-scan latency of a single recording (B = 1): device events around one call of one scan, after warm-up.
Prints one JSON line; nothing is written to the tree."""
from __future__ import annotations

import argparse
import importlib
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the numbers are reported without a card name rather than not at all
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fleets", default="132,1024")
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--latency-scans", type=int, default=200)
    a = ap.parse_args()
    import torch  # device events
    abi, synth = pkg.abi, pkg.synth
    P = pkg.load("plicp")
    laser = synth.Laser()
    pool_n = max(a.scans, a.latency_scans) + 64
    _, _, pool = synth.make_trajectory(3, pool_n, laser, step_xy=0.02, step_th_deg=0.5)
    pool = pool.astype(np.float32)
    fields = (float(np.float32(laser.min_angle)), float(np.float32(laser.angular_resolution)), 0.1, 30.0)
    params = abi.plicp_odom_params()
    res = {"card": None, "power_limit": None, "beams": laser.n_readings}

    def stamps(S):
        t = np.arange(S) * 100_000_000
        return np.stack([100 + t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)

    fleets = []
    for B in [int(x) for x in a.fleets.split(",")]:
        S = a.scans
        recs = [pool[b % 64: b % 64 + S] for b in range(B)]
        st = [stamps(S)] * B
        o = P.Odometry(params, B, laser.n_readings, *fields)
        o.process([r[:2] for r in recs], [s[:2] for s in st])  # warm-up
        o.reset()
        t0 = time.perf_counter()
        o.process(recs, st)
        dt = time.perf_counter() - t0
        o.close()
        fleets.append({"B": B, "S": S, "seconds": dt, "scans_per_s": B * S / dt})
    res["fleet"] = fleets
    o = P.Odometry(params, 1, laser.n_readings, *fields)
    st = stamps(a.latency_scans)
    o.process([pool[:1]], [st[:1]])
    ms = []
    for k in range(1, a.latency_scans):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        o.process([pool[k:k + 1]], [st[k:k + 1]])
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    o.close()
    ms = np.array(ms)
    res["latency_ms"] = {"median": float(np.median(ms)), "p10": float(np.percentile(ms, 10)),
                         "p90": float(np.percentile(ms, 90)), "scans": len(ms)}
    res["card"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
