"""Throughput of lesson3's scan-to-scan PL-ICP node on the device (b2s_plicp_scan_match_process), next to the lesson3
odometry node (b2s_plicp_odom_process) at the same shape.

  python tools/plicp_scan_match_bench.py [--shapes 1x1000,132x100,1024x100] [--repeats 3]

For each shape B x S, B recordings of S scans x 1081 beams (synthetic drives, synth.py, built from a pool of scans along
one trajectory; recording b starts at pool offset b % 64) go through ONE call of each handle: host ranges in, steps out,
timed with a host clock around the call (the call ends in a stream synchronise).  The scan-match node runs one CTA per
scan pair; the odometry node one CTA per recording.  Both start from fresh state (reset) after a two-scan warm-up call,
and the median of --repeats calls is reported, with the card's name and power limit read in the same run.  Also
checks that the scan-match results of the first recording equal a B = 1 handle's.  Prints one JSON line; nothing is
written to the tree."""
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
    ap.add_argument("--shapes", default="1x1000,132x100,1024x100")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-odometry", action="store_true")
    a = ap.parse_args()
    abi, synth = pkg.abi, pkg.synth
    P = pkg.load("plicp")
    M = pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    laser = synth.Laser()
    shapes = [tuple(int(v) for v in s.split("x")) for s in a.shapes.split(",")]
    pool_n = max(S for _, S in shapes) + 64
    _, _, pool = synth.make_trajectory(3, pool_n, laser, step_xy=0.02, step_th_deg=0.5)
    pool = pool.astype(np.float32)
    amin, ainc = np.float32(laser.min_angle), np.float32(laser.angular_resolution)
    fields = (float(amin), float(ainc), 0.1, 30.0)
    icp = abi.icp_params()
    res = {"card": None, "power_limit": None, "beams": laser.n_readings, "repeats": a.repeats, "shapes": []}

    def timed(fn):
        ts = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts)), float(min(ts)), float(max(ts)), out

    for B, S in shapes:
        recs = [pool[b % 64: b % 64 + S] for b in range(B)]
        lims = [np.tile(np.float32([0.1, 30.0]), (S, 1))] * B
        h = P.ScanMatch(icp, [laser.n_readings] * B, [amin] * B, [ainc] * B)
        h.process([r[:2] for r in recs], [l[:2] for l in lims])  # warm-up

        def sm():
            h.reset()
            return h.process(recs, lims)
        med, lo, hi, got = timed(sm)
        h.close()
        one = P.ScanMatch(icp, [laser.n_readings], [amin], [ainc])
        assert got[0].tobytes() == one.process([recs[0]], [lims[0]])[0].tobytes(), "fleet differs from B = 1"
        one.close()
        row = {"B": B, "S": S, "scan_match": {"seconds": med, "min": lo, "max": hi, "scans_per_s": B * S / med,
                                              "valid": float(np.mean(np.concatenate(got)["valid"][1:]))}}
        if not a.skip_odometry:
            st = np.stack([100 + np.arange(S) // 10, (np.arange(S) % 10) * 100_000_000], 1).astype(np.uint32)
            o = P.Odometry(abi.plicp_odom_params(icp=icp), B, laser.n_readings, *fields)
            o.process([r[:2] for r in recs], [st[:2]] * B)

            def od():
                o.reset()
                return o.process(recs, [st] * B)
            med, lo, hi, _ = timed(od)
            o.close()
            row["odometry"] = {"seconds": med, "min": lo, "max": hi, "scans_per_s": B * S / med}
        res["shapes"].append(row)
    res["card"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
