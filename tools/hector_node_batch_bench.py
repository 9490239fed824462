"""Time lesson4's Hector SLAM node handle with several nodes (b2s_hector_node_process_batch) against the same
recordings through one single-node handle each, called one after another.  Each node replays a seeded synthetic walk of
1081-beam scans (Hokuyo UTM-30LX geometry) at 40 Hz, starting at its own place in the walk, at the node's default
parameters (2048 x 2048 level 0, three levels).  Host ranges in, every published map handed to a callback on the host.

  python tools/hector_node_batch_bench.py [--scans 2000] [--batches 1,32,132]

Runs every batch size twice: with map_pub_period 2 s (a 4 MiB map per node every 80 scans: the copy back bounds the
call) and with 1e6 s (one publish per node: the matching bounds it).  Prints one JSON line with, per (B, period):
scans/s of the batched handle and of the sequential single-node handles, the maps handed out and the payload bytes
copied back, and the card's name and power limit, read in the same run.  It needs a CUDA device; there is no CPU
fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
from hector_node_bench import card  # noqa: E402


def recordings(B, n, laser):
    """B recordings of n scans: a 500-scan walk looped forwards and backwards, node b starting 37 b scans in, and its
    own start stamp (40 Hz)."""
    _, _, base = pkg.synth.make_trajectory(5, 500, laser, step_xy=0.02, step_th_deg=0.5)
    loop = np.concatenate([base, base[::-1]]).astype(np.float32)
    out = []
    for b in range(B):
        idx = (37 * b + np.arange(n)) % len(loop)
        t = (1_000 + b) * 1_000_000_000 + np.arange(n, dtype=np.int64) * 25_000_000
        st = np.stack([t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)
        out.append((np.ascontiguousarray(loop[idx]), st))
    return out


def run_batch(N, geom, recs, period):
    h = N.HectorNodeBatch([N.node_params(dict(map_pub_period=period))] * len(recs), geom,
                          [(0, 0, 0, 0, 0, 0, 1)] * len(recs))
    count = [0, 0]

    def on_map(b, m):
        count[0] += 1
        count[1] += m["payload"].nbytes
    t0 = time.perf_counter()
    h.process([r for r, _ in recs], [s for _, s in recs], on_map=on_map)
    s = time.perf_counter() - t0
    h.close()
    return s, count[0], count[1]


def run_sequential(N, geom, recs, period):
    s = 0.0
    for r, st in recs:
        node = N.HectorNode(N.node_params(dict(map_pub_period=period)), geom)
        t0 = time.perf_counter()
        node.process(r, st, on_map=lambda m: None)
        s += time.perf_counter() - t0
        node.close()
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=2000)
    ap.add_argument("--batches", default="1,32,132")
    a = ap.parse_args()
    M = pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("hector_node_batch_bench: no CUDA device (there is no CPU fallback)")
    N, R = pkg.load("hector_node"), pkg.load("rosio")
    laser = pkg.synth.Laser()
    amin, inc = np.float32(laser.min_angle), np.float32(laser.angular_resolution)
    geom = R.make_msg(amin, amin + inc * np.float32(laser.n_readings - 1), inc, np.float32(0.1), np.float32(30.0),
                      np.zeros(laser.n_readings, np.float32))
    batches = [int(b) for b in a.batches.split(",")]
    recs = recordings(max(batches), a.scans, laser)
    run_batch(N, geom, [(r[:100], s[:100]) for r, s in recs[:2]], 2.0)  # warm-up: module load, pools, pinned buffers
    rows = []
    for B in batches:
        for period in (2.0, 1e6):
            s, maps, nbytes = run_batch(N, geom, recs[:B], period)
            seq = run_sequential(N, geom, recs[:B], period)
            total = B * a.scans
            rows.append(dict(batch=B, map_pub_period=period, scans=total, s=round(s, 3), scans_per_s=round(total / s),
                             maps=maps, payload_bytes=nbytes, payload_gb_per_s=round(nbytes / s / 1e9, 2),
                             sequential_s=round(seq, 3), sequential_scans_per_s=round(total / seq),
                             speedup=round(seq / s, 2)))
    print(json.dumps(dict(scans_per_node=a.scans, beams=laser.n_readings, map="2048x2048, 3 levels", runs=rows,
                          kernel="k_hs_stream_batch<true, true> (one CTA per node, exact mode)", card=card())))


if __name__ == "__main__":
    main()
