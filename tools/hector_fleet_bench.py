"""Time a fleet of Hector SLAM processors replaying their recordings: one b2s_hector_slam_process_stream_batch call
(k_hs_stream_batch, one CTA per processor) against stepping the same streams scan by scan.

  python tools/hector_fleet_bench.py [--processors 128] [--scans 1000] [--worlds room,hall] [--modes exact,fast]
                                     [--out FILE]

Workload: B processors, each replaying its own self-driven synth.make_trajectory recording (1081-beam scans, 0.05 m /
1 degree steps) on a 1000 x 1000 x 3-level map at 0.05 m with the node defaults (0.4 / 0.9 update factors, 0.4 m /
0.9 rad gate), in the small room world and in the 44 m x 44 m hall with 24 boxes (30 m rays: heavy map updates).
For each world and mode it reports, in one JSON line:
  - fleet: the whole recording of every processor in one call, host arrays in, poses out (end to end, synchronised);
  - step_host: b2s_hector_slam_update_batch once per step (scans copied up and per-scan poses back each step);
  - step_device: b2s_hector_slam_update_batch_device once per step, the scans already on the device, no hints (each
    processor chains through its last scan-match pose), synchronised at the end;
  - scans/s end to end, the bytes each path copies, and the kernels' own time from torch.profiler in a separate pass;
  - whether the fleet's poses, gate decisions, last poses and every cell of every level equal the stepping's
    (bit for bit: the paths run the same match and map-update code);
  - the card's name and power limit, read in the same run.
It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = "creating-2d-laser-slam-from-scratch_b200"
pkg = importlib.import_module(PKG)
KW = dict(resolution=0.05, size_x=1000, size_y=1000, start=(0.5, 0.5), levels=3, update_free=0.4, update_occupied=0.9,
          min_dist=0.4, min_angle=0.9)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def recording(job):
    """(first pose, scans) of one processor: a seeded trajectory in the room or the hall, as level-0 map cells."""
    world, seed, n = job
    synth = pkg.synth
    to_cells = importlib.import_module(PKG + ".hector").scan_to_data_container
    laser = synth.Laser()
    if world == "hall":
        _, poses, ranges = synth.make_trajectory(seed, n, laser, half_w=22.0, half_h=22.0, step_xy=0.05, step_th_deg=1.0,
                                                 n_boxes=24)
    else:
        _, poses, ranges = synth.make_trajectory(seed, n, laser, step_xy=0.05, step_th_deg=1.0)
    return poses[0].astype(np.float32), [to_cells(ranges[i], laser, 0.05, max_dist=30.0, min_dist=0.2) for i in range(n)]


class Packed:
    """The fleet call's host arrays, built once so that the timed call is the library's own work."""

    def __init__(self, streams, firsts):
        self.B, self.n = len(streams), len(streams[0])
        self.ns = np.full(self.B, self.n, np.int32)
        scans = [s for st in streams for s in st]
        self.cnt = np.array([len(s) for s in scans], np.int32)
        self.cat = np.ascontiguousarray(np.concatenate(scans, 0), np.float32)
        self.firsts = np.ascontiguousarray(firsts, np.float32)
        self.poses = np.zeros((self.B * self.n, 3), np.float32)
        self.upd = np.zeros(self.B * self.n, np.int32)
        self.covs = np.zeros((self.B, 9), np.float32)
        self.origo = np.zeros(2, np.float32)

    def call(self, g):
        f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
        i = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))  # noqa: E731
        pkg.load("matcher").check(g.L.b2s_hector_slam_process_stream_batch(
            g.h, i(self.ns), f(self.cat), i(self.cnt), f(self.origo), f(self.firsts), None, 0, f(self.poses),
            i(self.upd), f(self.covs)))
        return self.poses.reshape(self.B, self.n, 3).copy(), self.upd.reshape(self.B, self.n).astype(bool)

    def h2d_bytes(self):
        return int(self.cat.nbytes + self.cnt.nbytes + 8 * len(self.cnt) + 16 * self.B + self.firsts.nbytes)

    def d2h_bytes(self):
        return 64 * len(self.cnt)


def same_state(a, b, B, levels):
    """last poses and every cell of every level of every processor, bit for bit"""
    for p in range(B):
        for x, y in zip(a.last_poses(p), b.last_poses(p)):
            if not np.array_equal(x.view(np.int32), y.view(np.int32)):
                return False
        for lvl in range(levels):
            (la, ua), (lb, ub) = a.level_of(p, lvl), b.level_of(p, lvl)
            if not (np.array_equal(ua, ub) and np.array_equal(la.view(np.int32), lb.view(np.int32))):
                return False
    return True


def kernel_ms(fn):
    """device time of the Hector kernels while fn runs, from torch.profiler (CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in ("k_hs_stream_batch", "k_hs_match", "k_hs_mark", "k_hs_apply"):
            if k in ev.key:
                out[k] = round(out.get(k, 0.0) + ev.device_time_total / 1e3, 3)
    return out


def run(H, streams, firsts, exact, cap):
    import torch
    B, n = len(streams), len(streams[0])
    kw = dict(KW, exact=exact)
    packed = Packed(streams, firsts)
    # warm-up on a throwaway handle: module loading and the first launches of every kernel the timed runs use
    w = H.HectorSlam(batch=B, max_points=cap, **kw)
    w.process_stream_batch([s[:2] for s in streams], (0, 0), first_hints=firsts)
    w.update_batch([s[2] for s in streams], (0, 0), None)
    w.close()
    torch.cuda.synchronize()

    gf = H.HectorSlam(batch=B, max_points=cap, **kw)
    t0 = time.perf_counter()
    pf, uf = packed.call(gf)
    t_fleet = time.perf_counter() - t0

    gs = H.HectorSlam(batch=B, max_points=cap, **kw)
    ps, us = np.zeros((B, n, 3), np.float32), np.zeros((B, n), bool)
    t0 = time.perf_counter()
    for i in range(n):
        p, _, u = gs.update_batch([s[i] for s in streams], (0, 0), firsts if i == 0 else None)
        ps[:, i], us[:, i] = p, u
    t_host = time.perf_counter() - t0

    dev = torch.device("cuda")
    pad = np.zeros((n, B, cap, 2), np.float32)
    cnt = np.zeros((n, B), np.int32)
    for b, s in enumerate(streams):
        for i, sc in enumerate(s):
            pad[i, b, :len(sc)] = sc
            cnt[i, b] = len(sc)
    d_pts, d_cnt = torch.from_numpy(pad).to(dev), torch.from_numpy(cnt).to(dev)
    d_first = torch.from_numpy(np.ascontiguousarray(firsts)).to(dev)
    max_n = [int(cnt[i].max()) for i in range(n)]
    del pad

    def step_device(g):
        for i in range(n):
            g.update_batch_device(d_pts[i].data_ptr(), d_cnt[i].data_ptr(), max_n[i], (0, 0),
                                  d_first.data_ptr() if i == 0 else None)
        g.sync()

    gd = H.HectorSlam(batch=B, max_points=cap, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    step_device(gd)
    t_dev = time.perf_counter() - t0

    equal_poses = bool(np.array_equal(pf.view(np.int32), ps.view(np.int32)) and np.array_equal(uf, us))
    equal_host = same_state(gf, gs, B, KW["levels"])
    equal_dev = same_state(gf, gd, B, KW["levels"])
    max_diff = float(np.nanmax(np.abs(pf - ps))) if pf.size else 0.0
    visits = gf.stats()["cell_visits"]
    for g in (gf, gs, gd):
        g.close()

    # kernel time in a pass of its own (the profiler slows the host side)
    prof = {}
    try:
        g = H.HectorSlam(batch=B, max_points=cap, **kw)
        prof["fleet"] = kernel_ms(lambda: packed.call(g))
        g.close()
        g = H.HectorSlam(batch=B, max_points=cap, **kw)
        prof["step_device"] = kernel_ms(lambda: step_device(g))
        g.close()
    except Exception as e:  # the end-to-end numbers stand on their own
        prof = {"error": repr(e)}
    del d_pts, d_cnt, d_first
    torch.cuda.empty_cache()

    scans = B * n
    step_h2d = n * B * (cap * 8 + 4) + B * 12  # padded rows and counts every step, the first hints once
    return {
        "scans": scans, "map_updates": int(uf.sum()), "cell_visits": int(visits),
        "fleet": {"s": round(t_fleet, 4), "scans_per_s": round(scans / t_fleet, 1),
                  "h2d_bytes": packed.h2d_bytes(), "d2h_bytes": packed.d2h_bytes()},
        "step_host": {"s": round(t_host, 4), "scans_per_s": round(scans / t_host, 1), "h2d_bytes": step_h2d,
                      "d2h_bytes": 64 * B * n},
        "step_device": {"s": round(t_dev, 4), "scans_per_s": round(scans / t_dev, 1), "h2d_bytes": 0, "d2h_bytes": 0,
                        "note": "scans uploaded before the timed loop (not counted); nothing returned per step"},
        "fleet_over_step_host": round(t_host / t_fleet, 3), "fleet_over_step_device": round(t_dev / t_fleet, 3),
        "kernel_ms": prof,
        "fleet_equals_step_host": equal_poses and equal_host, "fleet_equals_step_device": equal_dev,
        "fleet_vs_step_host_max_abs_pose_diff": max_diff,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--processors", type=int, default=128)
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--worlds", default="room,hall")
    ap.add_argument("--modes", default="exact,fast")
    ap.add_argument("--seed", type=int, default=5000)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    H, M = pkg.load("hector"), pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("hector_fleet_bench: no CUDA device")
    # the recordings first, in worker processes that never touch the device
    recs = {}
    for world in a.worlds.split(","):
        t0 = time.perf_counter()
        jobs = [(world, a.seed + 1000 * (world == "hall") + b, a.scans) for b in range(a.processors)]
        with ProcessPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
            recs[world] = (list(ex.map(recording, jobs)), time.perf_counter() - t0)
    import torch
    torch.cuda.init()
    result = {"workload": f"{a.processors} Hector processors x {a.scans} self-driven scans each (1081 beams), "
                          "1000 x 1000 x 3-level maps at 0.05 m, node defaults",
              "card": card(), "device": torch.cuda.get_device_name(0), "worlds": {}}
    for world, (rec, secs) in recs.items():
        firsts = np.stack([r[0] for r in rec])
        streams = [r[1] for r in rec]
        cap = max(len(s) for st in streams for s in st)
        entry = {"points_per_scan_mean": round(float(np.mean([len(s) for st in streams for s in st])), 1),
                 "max_points": cap, "recordings_s": round(secs, 1)}
        for mode in a.modes.split(","):
            entry[mode] = run(H, streams, firsts, mode == "exact", cap)
        result["worlds"][world] = entry
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
