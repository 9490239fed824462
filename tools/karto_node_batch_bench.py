"""Time many lesson6 Karto SLAM nodes in one handle (b2s_karto_node_create_batch) against the same nodes as single
handles called one after another: B seeded hall recordings (a robot circling a 9 m radius in a 28 m x 24 m hall with 12
boxes, synth.make_loop_trajectory, one seed per node, 1081 beams, 10 Hz) x S scans at the shipped
config/mapper_params.yaml values (tests/karto_node_cases.SHIPPED_YAML) with the node's default 5 s map interval.

  python tools/karto_node_batch_bench.py [--batches 1,32,132] [--scans 300] [--single-scans 3000] [--dry-run]

Prints one JSON line per B:
  - batch_s, scans_per_s, key_frames_per_s: all B recordings in one b2s_karto_node_process_batch call, end to end;
  - singles_s, singles_scans_per_s, speedup: the same recordings through B single handles in turn;
  - rounds, match_launches, matches, maps, match_s, map_s, map_share, map_bytes_d2h: b2s_karto_node_last_timing of
    the batched call (where its wall time went; map_share = map_s / batch_s);
  - equal: every node's states, poses and maps equal its single handle's;
then, unless --single-scans 0, one line re-measuring one node on a --single-scans recording (the single-node bench's
workload, tools/karto_node_bench.py) through the batch-of-one handle.  Each line carries the card's name and power
limit, read in the same run.  It needs a CUDA device; there is no CPU fallback.  --dry-run checks the arguments and
builds the recordings without a device.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def recordings(B, S, step=0.25):
    import karto_node_cases as kc
    laser = kc.pkg.synth.Laser(type=0, n_readings=kc.N_BEAMS, min_angle=float(kc.ANGLE_MIN),
                               max_angle=float(kc.ANGLE_MIN + kc.N_BEAMS * kc.ANGLE_INC),
                               angular_resolution=float(kc.ANGLE_INC), range_threshold=12.0)
    out = []
    for b in range(B):
        _, _, odom, ranges = kc.pkg.synth.make_loop_trajectory(11 + b, S, laser, radius=9.0, step=step, half_w=14.0,
                                                               half_h=12.0, n_boxes=12)
        out.append((ranges.astype(np.float32), kc.stamps_10hz(S), kc.odom_rows(odom)))
    return out


def params_and_geometry(S):
    import karto_node_cases as kc
    prm, _ = KN.node_params(dict(kc.SHIPPED_YAML))
    prm.map_update_interval = 5.0
    c = kc.Case("bench", dict(kc.SHIPPED_YAML), np.zeros((1, kc.N_BEAMS), np.float32), kc.stamps_10hz(1),
                np.zeros((1, 7)))
    return prm, c.geometry(), c.mount


def run_batch(prm, geom, mount, recs):
    B = len(recs)
    fleet = KN.KartoNodeBatch([prm] * B, geom, [mount] * B)
    t0 = time.perf_counter()
    got = fleet.process([r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs])
    dt = time.perf_counter() - t0
    timing = fleet.last_timing()
    fleet.close()
    return dt, got, timing


def run_singles(prm, geom, mount, recs):
    outs, dt = [], 0.0
    for r in recs:
        node = KN.KartoNode(prm, geom, mount)
        t0 = time.perf_counter()
        outs.append(node.process(r[0], r[1], r[2]))
        dt += time.perf_counter() - t0
        node.close()
    return dt, outs


def same(a, b):
    return (np.array_equal(a["state"], b["state"]) and np.array_equal(a["pose"], b["pose"]) and
            len(a["maps"]) == len(b["maps"]) and
            all(x[0] == y[0] and np.array_equal(x[2], y[2]) for x, y in zip(a["maps"], b["maps"])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,32,132")
    ap.add_argument("--scans", type=int, default=300)
    ap.add_argument("--single-scans", type=int, default=3000)
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args()
    batches = [int(x) for x in a.batches.split(",") if x]
    if not batches or min(batches) < 1 or max(batches) > 1024 or a.scans < 1 or a.single_scans < 0:
        ap.error("--batches must be 1..1024, --scans >= 1, --single-scans >= 0")
    prm, geom, mount = params_and_geometry(a.scans)
    recs = recordings(max(batches), a.scans)
    if a.dry_run:
        print(json.dumps(dict(batches=batches, scans=a.scans, recordings=len(recs), beams=int(recs[0][0].shape[1]))))
        return
    who = card()
    run_batch(prm, geom, mount, recs[:2])  # warm-up: the CUDA context and the kernels' first launches
    for B in batches:
        part = recs[:B]
        batch_s, got, t = run_batch(prm, geom, mount, part)
        singles_s, want = run_singles(prm, geom, mount, part)
        scans = B * a.scans
        key = int(sum((g["state"] == KN.PROCESSED).sum() for g in got))
        print(json.dumps(dict(batch=B, scans=a.scans, beams=int(part[0][0].shape[1]), key_frames=key,
                              batch_s=round(batch_s, 3), scans_per_s=round(scans / batch_s, 1),
                              key_frames_per_s=round(key / batch_s, 1), singles_s=round(singles_s, 3),
                              singles_scans_per_s=round(scans / singles_s, 1), speedup=round(singles_s / batch_s, 2),
                              rounds=int(t["rounds"]), match_launches=int(t["match_launches"]),
                              matches=int(t["matches"]), maps=int(t["maps"]), match_s=round(t["match_s"], 3),
                              map_s=round(t["map_s"], 3), map_share=round(t["map_s"] / batch_s, 3),
                              map_bytes_d2h=int(t["map_bytes_d2h"]),
                              equal=all(same(g, w) for g, w in zip(got, want)), card=who)), flush=True)
    if a.single_scans:
        rec = recordings(1, a.single_scans)
        s, got, t = run_batch(prm, geom, mount, rec)
        key = int((got[0]["state"] == KN.PROCESSED).sum())
        print(json.dumps(dict(batch=1, scans=a.single_scans, key_frames=key, batch_s=round(s, 3),
                              scans_per_s=round(a.single_scans / s, 1), key_frames_per_s=round(key / s, 1),
                              rounds=int(t["rounds"]), maps=int(t["maps"]), match_s=round(t["match_s"], 3),
                              map_s=round(t["map_s"], 3), map_share=round(t["map_s"] / s, 3), card=who)), flush=True)


if __name__ == "__main__":
    main()
