"""Time lesson2's ICP on a whole recording: b2s_pcl_icp_align over the consecutive pairs of a seeded synthetic recording
(1081-beam Hokuyo UTM-30LX scans, node defaults: 10 iterations, invalid readings kept as origin points).

  python tools/pcl_icp_bench.py [--scans 10000] [--warmup 2] [--repeats 5] [--cpu-pairs 20] [--out DIR]

Prints one JSON line:
  - end_to_end_ms: host ranges in, results out, synchronised (median and spread of the repeats);
  - kernel_ms / kernel_us_per_pair: device time of the conversion and ICP kernels from torch.profiler (a separate run,
    so the profiler does not slow the timed ones); copies and allocation are the rest of end_to_end_ms;
  - cpu_ms_per_pair: the C restatement on one core, over the first --cpu-pairs pairs;
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=10000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-pairs", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="directory for the profiler trace")
    a = ap.parse_args()

    abi, synth = pkg.abi, pkg.synth
    P, M = pkg.load("pcl_icp"), pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("pcl_icp_bench: no CUDA device")
    laser = synth.Laser()
    _, _, ranges = synth.make_trajectory(a.seed, a.scans, laser, step_xy=0.05, step_th_deg=1.0)
    rng = np.random.default_rng(a.seed)
    drop = rng.random(ranges.shape) < 0.01  # 1 % NaN readings: the node keeps them as origin points
    ranges[drop] = np.nan
    r = np.ascontiguousarray(ranges, np.float32)
    amin, inc = np.float32(laser.min_angle), np.float32(laser.angular_resolution)
    params = abi.pcl_icp_params()
    n_pairs = a.scans - 1

    for _ in range(a.warmup):
        P.align(params, r, amin, inc, 0.1, 30.0)
    times = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        res = P.align(params, r, amin, inc, 0.1, 30.0)
        times.append((time.perf_counter() - t0) * 1e3)

    # kernel time, in a run of its own
    kernel = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            P.align(params, r, amin, inc, 0.1, 30.0)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if "k_pcl_" in ev.key:
                name = "k_pcl_icp" if "k_pcl_icp" in ev.key else "k_pcl_cloud"
                kernel[name] = kernel.get(name, 0.0) + ev.device_time_total / 1e3
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.out, "pcl_icp.pt.trace.json"))
    except Exception as e:  # the end-to-end numbers stand on their own
        kernel = {"error": repr(e)}

    from oracle import pcl_icp_port as port
    k = min(a.cpu_pairs, n_pairs)
    t0 = time.perf_counter()
    for i in range(k):
        c = port.pcl_icp_align(params, r[i], r[i + 1], amin, inc, 0.1, 30.0)
        assert res[i]["iterations"] == c.iterations and res[i]["fitness_score"] == c.fitness_score, i
    cpu_ms = (time.perf_counter() - t0) * 1e3 / max(k, 1)

    med = statistics.median(times)
    icp_ms = kernel.get("k_pcl_icp") if isinstance(kernel.get("k_pcl_icp"), float) else None
    print(json.dumps({
        "workload": f"lesson2 ICP, {a.scans} scans x 1081 beams, {n_pairs} consecutive pairs, node defaults",
        "card": card(),
        "end_to_end_ms": {"median": round(med, 3), "min": round(min(times), 3), "max": round(max(times), 3),
                          "repeats": a.repeats},
        "pairs_per_s": round(n_pairs / (med / 1e3), 1),
        "kernel_ms": {k2: round(v, 3) for k2, v in kernel.items()} if "error" not in kernel else kernel,
        "kernel_us_per_pair": round(icp_ms * 1e3 / n_pairs, 3) if icp_ms else None,
        "iterations_mean": float(np.mean(res["iterations"])),
        "converged": int(res["converged"].sum()),
        "cpu_ms_per_pair": round(cpu_ms, 3),
        "cpu_pairs_timed": k,
    }))


if __name__ == "__main__":
    main()
