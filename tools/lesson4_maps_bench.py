"""Time lesson4's make-map nodes on a whole recording: b2s_gmapping_node_maps and b2s_hector_mapping_node_maps over a
seeded synthetic recording of 1081-beam scans (Hokuyo UTM-30LX geometry, 2 % NaN / inf / 0 dropouts) at the nodes'
default parameters (1599 x 1599 maps, 2.56 MB per scan), host ranges in, maps out into one page-locked buffer reused
chunk by chunk.

  python tools/lesson4_maps_bench.py [--scans 1000] [--chunk 100] [--warmup 2] [--repeats 5] [--out DIR]

Prints one JSON line per node:
  - end_to_end_ms / scans_per_s: the whole recording, host ranges in, maps on the host (median, min, max of the repeats);
  - kernel_ms: device time of the call's kernels from torch.profiler, in a run of its own, and the device-to-host copy
    time it lists; copy_share = that copy time over the profiled call's device span;
  - bytes_back: payload bytes copied to the host;
  - today_ms_per_scan (GMapping only): the route through the per-scan handle, b2s_gmap_create + compute_map + copy_ros +
    destroy with the beam cache on the host, over the first --today-scans scans;
  - cpu_ms_per_scan: the C restatement on one core over the first --cpu-scans scans;
  - the card's name and power limit, read in the same run.
It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import re
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


def whole(fn, r, fields, buf, chunk):
    """The recording in chunks of `chunk` scans through one page-locked buffer."""
    for s in range(0, len(r), chunk):
        k = min(chunk, len(r) - s)
        fn(r[s:s + k], fields, out=buf[:k])


def profile_call(fn, r, fields, buf, chunk, name, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        whole(fn, r, fields, buf, chunk)
        torch.cuda.synchronize()
    kernels, copy_ms, t0, t1 = {}, 0.0, None, None
    for ev in prof.events():
        if ev.device_type is None or str(ev.device_type) != "DeviceType.CUDA":
            continue
        start, end = ev.time_range.start, ev.time_range.end
        t0 = start if t0 is None else min(t0, start)
        t1 = end if t1 is None else max(t1, end)
        kern = re.search(r"\b(k_\w+)", ev.name)
        if kern:
            kernels[kern.group(1)] = kernels.get(kern.group(1), 0.0) + (end - start) / 1e3
        elif "DtoH" in ev.name:
            copy_ms += (end - start) / 1e3
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"lesson4_{name}.pt.trace.json"))
    span = (t1 - t0) / 1e3 if t0 is not None else float("nan")
    return kernels, copy_ms, span


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--chunk", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-scans", type=int, default=20)
    ap.add_argument("--today-scans", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    a = ap.parse_args()

    NM, M = pkg.load("node_maps"), pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("lesson4_maps_bench: no CUDA device")
    import torch
    from oracle import lesson4_nodes_port as port
    synth = pkg.synth
    laser = synth.Laser()
    _, _, ranges = synth.make_trajectory(a.seed, a.scans, laser, step_xy=0.05, step_th_deg=1.0)
    rng = np.random.default_rng(a.seed)
    m = rng.random(ranges.shape)
    ranges[m < 0.01] = np.nan
    ranges[(m >= 0.01) & (m < 0.015)] = np.inf
    ranges[(m >= 0.015) & (m < 0.02)] = 0.0
    r = np.ascontiguousarray(ranges, np.float32)
    fields = (np.float32(laser.min_angle), np.float32(laser.angular_resolution), np.float32(0.1), np.float32(30.0))
    c = card()
    for name, fn in (("gmapping", NM.gmapping_maps), ("hector", NM.hector_maps)):
        w, h = (port.gmapping_dims if name == "gmapping" else port.hector_dims)(
            NM.gmapping_params() if name == "gmapping" else NM.hector_params())
        chunk = min(a.chunk, len(r))
        buf = torch.empty((chunk, h, w), dtype=torch.int8, pin_memory=True).numpy()
        for _ in range(a.warmup):
            whole(fn, r, fields, buf, chunk)
        times = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            whole(fn, r, fields, buf, chunk)
            times.append((time.perf_counter() - t0) * 1e3)
        try:
            kernels, copy_ms, span = profile_call(fn, r, fields, buf, chunk, name, a.out)
        except Exception as e:  # the end-to-end numbers stand on their own
            kernels, copy_ms, span = {"error": repr(e)}, float("nan"), float("nan")

        k = min(a.cpu_scans, len(r))
        t0 = time.perf_counter()
        want = port.gmapping(fields, NM.gmapping_params(), r[:k])[0] if name == "gmapping" else \
            port.hector(fields, NM.hector_params(), r[:k])
        cpu_ms = (time.perf_counter() - t0) * 1e3 / max(k, 1)
        got = fn(r[:k], fields)
        assert np.array_equal(got, want), f"{name}: the device maps differ from the restatement"

        today = None
        if name == "gmapping":
            G = pkg.load("gmapping")
            kt = min(a.today_scans, len(r))
            # CreateCache on the host: the float angle, widened
            ang = (fields[0] + np.arange(r.shape[1], dtype=np.float32) * fields[1]).astype(np.float64)
            t0 = time.perf_counter()
            for s in range(kt):
                g = G.GMap()
                g.compute_map(r[s].astype(np.float64), ang)
                g.ros_map()
                g.close()
            today = (time.perf_counter() - t0) * 1e3 / max(kt, 1)

        med = statistics.median(times)
        print(json.dumps({
            "workload": f"lesson4 {name} node maps: {len(r)} scans x {r.shape[1]} beams, node defaults "
                        f"({w} x {h}), chunks of {chunk} into one page-locked buffer",
            "card": c,
            "end_to_end_ms": {"median": round(med, 2), "min": round(min(times), 2), "max": round(max(times), 2),
                              "repeats": a.repeats},
            "scans_per_s": round(len(r) / (med / 1e3), 1),
            "bytes_back": int(len(r)) * w * h,
            "kernel_ms": {k2: round(v, 3) for k2, v in kernels.items()} if "error" not in kernels else kernels,
            "copy_back_ms": round(copy_ms, 3),
            "profiled_device_span_ms": round(span, 3),
            "copy_share": round(copy_ms / span, 3) if span == span and span > 0 else None,
            "today_ms_per_scan": None if today is None else round(today, 3),
            "cpu_ms_per_scan": round(cpu_ms, 3),
            "cpu_scans_timed": k,
        }), flush=True)


if __name__ == "__main__":
    main()
