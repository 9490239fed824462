"""Time lesson1's corner picker on a whole recording: b2s_feature_detect over a seeded synthetic recording of 1081-beam
scans (Hokuyo UTM-30LX geometry, 2 % NaN / inf dropouts), host ranges in, picks, counts and curvature out.

  python tools/feature_bench.py [--scans 10000] [--warmup 2] [--repeats 5] [--cpu-scans 300] [--out DIR]

Two workloads, because the device's selection depends on the input:
  - natural: the synthetic scans as cast, whose sector cuts are decided by rank counting;
  - tied: the same scans rounded to half metres, so that most sector cuts are tied (tied_sectors gives the share) and
    one lane per such sector sorts it with the restated introsort.
Prints one JSON line per workload:
  - end_to_end_ms: host ranges in, results out, synchronised (median, min, max of the repeats);
  - kernel_ms: device time of k_feature_detect from torch.profiler, in a run of its own;
  - cpu_ms_per_scan: the C++ restatement (std::sort, as the node) on one core, over the first --cpu-scans scans;
  - tied_sectors: the share of sectors whose cut is tied (from the restatement);
  - the card's name and power limit, read in the same run.
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
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(name, r, a, F, fp, device_card):
    for _ in range(a.warmup):
        F.detect(r)
    times = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        got, cnt, curv = F.detect(r)
        times.append((time.perf_counter() - t0) * 1e3)

    kernel = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            F.detect(r)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if "k_feature_detect" in ev.key:
                kernel["k_feature_detect"] = kernel.get("k_feature_detect", 0.0) + ev.device_time_total / 1e3
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.out, f"feature_{name}.pt.trace.json"))
    except Exception as e:  # the end-to-end numbers stand on their own
        kernel = {"error": repr(e)}

    k = min(a.cpu_scans, len(r))
    want = fp.detect(r[:k])
    assert np.array_equal(got[:k].view(np.int32), want.ranges.view(np.int32)) and np.array_equal(cnt[:k], want.count)
    cpu_ms = fp.detect_timed(r[:k]) * 1e3 / max(k, 1)
    tied = float(np.mean([bin(int(t)).count("1") / 6.0 for t in want.tied]))

    med = statistics.median(times)
    print(json.dumps({
        "workload": f"lesson1 corner picks, {name}: {len(r)} scans x {r.shape[1]} beams, edge_threshold 1.0",
        "card": device_card,
        "end_to_end_ms": {"median": round(med, 3), "min": round(min(times), 3), "max": round(max(times), 3),
                          "repeats": a.repeats},
        "scans_per_s": round(len(r) / (med / 1e3), 1),
        "bytes_each_way": int(r.nbytes),
        "kernel_ms": {k2: round(v, 3) for k2, v in kernel.items()} if "error" not in kernel else kernel,
        "picks_mean": float(np.mean(cnt)),
        "tied_sectors": round(tied, 4),
        "cpu_ms_per_scan": round(cpu_ms, 4),
        "cpu_scans_timed": k,
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=10000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-scans", type=int, default=300)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    a = ap.parse_args()

    F, M = pkg.load("features"), pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("feature_bench: no CUDA device")
    from oracle import features_port as fp
    synth = pkg.synth
    laser = synth.Laser()
    _, _, ranges = synth.make_trajectory(a.seed, a.scans, laser, step_xy=0.05, step_th_deg=1.0)
    rng = np.random.default_rng(a.seed)
    m = rng.random(ranges.shape)
    ranges[m < 0.01] = np.nan
    ranges[(m >= 0.01) & (m < 0.02)] = np.inf
    natural = np.ascontiguousarray(ranges, np.float32)
    tied = np.ascontiguousarray(np.round(natural * 2.0) / 2.0, np.float32)
    c = card()
    run("natural", natural, a, F, fp, c)
    run("tied", tied, a, F, fp, c)


if __name__ == "__main__":
    main()
