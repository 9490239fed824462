"""Per-kernel timing of one CorrelateScan step at bench.py's cfg-2 shape (1024 matches, 1081 beams, 31 x 31 x 181,
0.05 m grid), from a torch.profiler CUDA trace (not a test).

Prints, per matcher kernel launch of a step in launch order, its mean duration over the profiled steps (a kernel
launched twice in a step, e.g. k_sweep_window in a pruned sweep, is listed twice), the step's last_pruned_frac() and
empty_window_frac, and the card name and power limit.  The trace and a JSON copy of the table go to --out.

usage: python tools/matcher_stage_profile.py [--out DIR] [--batch 1024] [--steps 10] [--warmup 3]"""
import argparse
import importlib
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
import torch  # noqa: E402

D = math.pi / 180


def short_name(name):
    name = name.split("(")[0]
    for pre in ("void ", "b2s::"):
        name = name.replace(pre, "")
    return name.strip()


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return repr(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    out_dir = args.out or tempfile.mkdtemp(prefix="matcher_stage_profile_")
    os.makedirs(out_dir, exist_ok=True)

    abi, synth = pkg.abi, pkg.synth
    M = pkg.load("matcher")
    B = args.batch
    cases = [synth.make_match_case(1_000_000 + i) for i in range(B)]  # bench.py's cfg-2 workload, rank 0
    ranges = np.stack([c.ranges for c in cases])
    poses = np.stack([c.odom_pose for c in cases])
    bran = np.stack([c.base_ranges for c in cases])[:, None, :]
    bpos = np.stack([c.base_pose for c in cases])[:, None, :]
    params, laser = abi.matcher_params(1.5, 0.05, 0.03, 9.25), abi.laser_from(synth.Laser())
    m = M.ScanMatcher(params, laser, max_batch=B, max_base_scans=1)
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m.set_scans(ranges, poses)
    m.add_scans(bran, bpos)
    for _ in range(args.warmup):
        m.correlate_scan(poses, se)
    m.sync()

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            m.correlate_scan(poses, se)  # synchronous: returns with the results on the host
    trace = os.path.join(out_dir, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel" and "k_" in e.get("name", "")),
                     key=lambda e: e["ts"])
    # split into steps: every step starts with k_bases
    steps, cur = [], None
    for e in kernels:
        nm = short_name(e["name"])
        if nm == "k_bases":
            cur = []
            steps.append(cur)
        if cur is not None:
            cur.append((nm, float(e["dur"]) * 1e-3, float(e["ts"]) * 1e-3))
    seqs = {tuple(n for n, _, _ in s) for s in steps}
    assert len(steps) == args.steps and len(seqs) == 1, (len(steps), seqs)
    names = list(next(iter(seqs)))
    dur = np.array([[d for _, d, _ in s] for s in steps])
    span = np.array([s[-1][2] + s[-1][1] - s[0][2] for s in steps])
    t = m.last_timing()
    res = {
        "card": torch.cuda.get_device_name(), "power_limit": power_limit(), "batch": B, "steps": args.steps,
        "kernels": [{"name": n, "mean_ms": float(dur[:, i].mean()), "min_ms": float(dur[:, i].min()),
                     "max_ms": float(dur[:, i].max())} for i, n in enumerate(names)],
        "kernel_sum_ms": float(dur.sum(axis=1).mean()), "first_to_last_kernel_ms": float(span.mean()),
        "last_pruned_frac": m.last_pruned_frac(), "empty_window_frac": m.last_stats()["empty_window_frac"],
        "stage_ms_last_step": {"lut": t["lut_ms"], "sweep": t["sweep_ms"], "reduce": t["reduce_ms"]},
    }
    m.close()
    with open(os.path.join(out_dir, "stage_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"card: {res['card']}, power limit: {res['power_limit']}, batch {B}, {args.steps} steps")
    print(f"{'#':>3} {'kernel':<32} {'mean ms':>9} {'min':>9} {'max':>9}")
    for i, k in enumerate(res["kernels"]):
        print(f"{i:>3} {k['name']:<32} {k['mean_ms']:9.4f} {k['min_ms']:9.4f} {k['max_ms']:9.4f}")
    print(f"    {'sum of kernels':<32} {res['kernel_sum_ms']:9.4f}")
    print(f"    {'first kernel start to last end':<32} {res['first_to_last_kernel_ms']:9.4f}")
    print(f"last_pruned_frac: {res['last_pruned_frac']!r}  empty_window_frac: {res['empty_window_frac']!r}")
    print(f"stage_ms (last step): {res['stage_ms_last_step']}")
    print(f"written to {out_dir}")


if __name__ == "__main__":
    main()
