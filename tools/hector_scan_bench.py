"""Time a Hector SLAM fleet replaying raw LaserScan recordings, end to end, two ways in the same run (alternating):
  (a) host:   b2s_ros_hector_scans converts every scan on the host (one call over the whole fleet), then
              b2s_hector_slam_process_stream_batch replays the points;
  (b) device: b2s_hector_slam_process_scans_batch uploads the float32 ranges and converts each scan inside the fleet
              kernel (k_hs_stream_batch<_, true>).

  python tools/hector_scan_bench.py [--processors 128] [--scans 1000] [--worlds room,hall] [--modes exact,fast]
                                    [--repeats 2] [--out FILE]

Workload: the recordings of tools/hector_fleet_bench.py (B processors, self-driven synth.make_trajectory walks, 1081-beam
scans, 0.05 m / 1 degree steps, 1000 x 1000 x 3-level maps at 0.05 m, node defaults), kept as float32 ranges; the
conversion uses the lesson4 node's defaults (projectLaser cutoff 30 m, use_max_scan_range 20 m, 0.2 - 30 m window,
laser at the base_link origin).  For each world and mode it reports, in one JSON line:
  - each arm's end-to-end seconds and scans/s (median over the repeats; host arrays in, poses out, synchronised), and
    for (a) the host conversion's share;
  - the device time of each call from CUDA events on the handle's stream (uploads + kernel + read-back) and the kernel's
    own time from torch.profiler in a separate pass;
  - the bytes each arm copies host -> device;
  - whether (a) and (b) give identical poses, gate flags, last Hessians, last poses, every cell of every level and
    kept-beam counts (bit for bit);
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
    """(first pose, float32 ranges [n, 1081]) of one processor, the trajectories of tools/hector_fleet_bench.py."""
    world, seed, n = job
    synth = pkg.synth
    laser = synth.Laser()
    if world == "hall":
        _, poses, ranges = synth.make_trajectory(seed, n, laser, half_w=22.0, half_h=22.0, step_xy=0.05, step_th_deg=1.0,
                                                 n_boxes=24)
    else:
        _, poses, ranges = synth.make_trajectory(seed, n, laser, step_xy=0.05, step_th_deg=1.0)
    return poses[0].astype(np.float32), ranges.astype(np.float32)


def kernel_ms(fn):
    """device time of k_hs_stream_batch while fn runs, from torch.profiler (CUDA activities): each arm runs one of its
    instantiations, <_, false> for (a) and <_, true> for (b)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    return round(sum(ev.device_time_total for ev in prof.key_averages() if "k_hs_stream_batch" in ev.key) / 1e3, 3)


def same_state(a, b, B, levels):
    for p in range(B):
        for x, y in zip(a.last_poses(p), b.last_poses(p)):
            if not np.array_equal(x.view(np.int32), y.view(np.int32)):
                return False
        for lvl in range(levels):
            (la, ua), (lb, ub) = a.level_of(p, lvl), b.level_of(p, lvl)
            if not (np.array_equal(ua, ub) and np.array_equal(la.view(np.int32), lb.view(np.int32))):
                return False
    return True


class Fleet:
    """Host arrays of both arms, built once so that a timed call is the library's own work."""

    def __init__(self, R, ranges, firsts):
        self.B, self.n, self.nr = ranges.shape
        self.ranges = np.ascontiguousarray(ranges.reshape(-1, self.nr))
        self.firsts = np.ascontiguousarray(firsts, np.float32)
        laser = pkg.synth.Laser()
        amin, inc = np.float32(laser.min_angle), np.float32(laser.angular_resolution)
        self.geom = R.make_msg(amin, amin + inc * np.float32(self.nr - 1), inc, 0.1, 30.0, np.zeros(self.nr, np.float32))
        self.filt = R.hector_scan_filter()  # the node's defaults, laser at the base_link origin
        self.scale = np.float32(1.0) / np.float32(KW["resolution"])
        T = self.B * self.n
        self.ns = np.full(self.B, self.n, np.int32)
        self.pts = np.zeros((T * self.nr, 2), np.float32)
        self.cnt = np.zeros(T, np.int32)
        self.kept = np.zeros(T, np.int32)
        self.origo = np.zeros(2, np.float32)
        self.poses, self.upd, self.covs = np.zeros((T, 3), np.float32), np.zeros(T, np.int32), np.zeros((self.B, 9), np.float32)
        R.hector_scans(self.geom, self.ranges[:1], self.filt, self.scale)  # binds the argument types
        self.L = pkg.load("matcher").lib()
        self.check = pkg.load("matcher").check

    @staticmethod
    def _f(a):
        return a.ctypes.data_as(C.POINTER(C.c_float))

    @staticmethod
    def _i(a):
        return a.ctypes.data_as(C.POINTER(C.c_int32))

    def host_arm(self, g, before_call=lambda: None):
        """(a): returns (seconds of the host conversion, seconds of the whole arm)"""
        f, i = self._f, self._i
        t0 = time.perf_counter()
        self.check(self.L.b2s_ros_hector_scans(C.byref(self.geom), C.byref(self.filt), self.scale, self.B * self.n,
                                               f(self.ranges), f(self.pts), i(self.cnt), f(self.origo)))
        t1 = time.perf_counter()
        before_call()
        self.check(g.L.b2s_hector_slam_process_stream_batch(g.h, i(self.ns), f(self.pts), i(self.cnt), f(self.origo),
                                                            f(self.firsts), None, 0, f(self.poses), i(self.upd),
                                                            f(self.covs)))
        t2 = time.perf_counter()
        return t1 - t0, t2 - t0

    def device_arm(self, g, before_call=lambda: None):
        f, i = self._f, self._i
        t0 = time.perf_counter()
        before_call()
        self.check(g.L.b2s_hector_slam_process_scans_batch(g.h, C.byref(self.geom), C.byref(self.filt), i(self.ns),
                                                           f(self.ranges), f(self.firsts), None, 0, f(self.poses),
                                                           i(self.upd), f(self.covs), i(self.kept)))
        return time.perf_counter() - t0

    def result(self):
        return self.poses.copy(), self.upd.copy(), self.covs.copy()

    def h2d_host_arm(self):  # points, counts, 64-bit offsets, first[B][2], first hints
        return int(8 * int(self.cnt.sum()) + 4 * len(self.cnt) + 8 * len(self.cnt) + 16 * self.B + self.firsts.nbytes)

    def h2d_device_arm(self):  # ranges, unit vectors, the ingest descriptor, B filters and origos, first[B][2], first hints
        return int(self.ranges.nbytes + 16 * self.nr + 40 + (128 + 8) * self.B + 16 * self.B + self.firsts.nbytes)


def run(H, R, ranges, firsts, exact, repeats):
    import torch
    B, n, nr = ranges.shape
    kw = dict(KW, exact=exact)
    fl = Fleet(R, ranges, firsts)
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    # warm-up of both kernels on a throwaway handle
    w = H.HectorSlam(batch=B, max_points=nr, stream=sp, **kw)
    w.process_scans_batch(fl.geom, [r[:2] for r in ranges], fl.filt, first_hints=firsts)
    w.process_stream_batch([[np.zeros((4, 2), np.float32)]] * B, (0, 0))
    w.close()
    torch.cuda.synchronize()

    times = {"host": [], "host_convert": [], "device": [], "host_event_ms": [], "device_event_ms": []}
    equal, last = True, {}
    for rep in range(repeats):
        for arm in ("host", "device"):  # alternating in the same run
            g = H.HectorSlam(batch=B, max_points=nr, stream=sp, **kw)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            mark = lambda: e0.record(stream)  # noqa: E731  (the events bracket the library call's device work)
            if arm == "host":
                tc, t = fl.host_arm(g, mark)
                times["host_convert"].append(tc)
            else:
                t = fl.device_arm(g, mark)
            e1.record(stream)
            e1.synchronize()
            times[arm].append(t)
            times[arm + "_event_ms"].append(e0.elapsed_time(e1))
            if rep == repeats - 1:
                last[arm] = (g, fl.result())
            else:
                g.close()
    (ga, (pa, ua, ca)), (gb, (pb, ub, cb)) = last["host"], last["device"]
    equal = bool(np.array_equal(pa.view(np.int32), pb.view(np.int32)) and np.array_equal(ua, ub)
                 and np.array_equal(ca.view(np.int32), cb.view(np.int32)) and np.array_equal(fl.kept, fl.cnt)
                 and same_state(ga, gb, B, KW["levels"]))
    updates = int(ua.sum())
    ga.close(), gb.close()

    prof = {}
    try:
        g = H.HectorSlam(batch=B, max_points=nr, stream=sp, **kw)
        prof["host"] = kernel_ms(lambda: fl.host_arm(g))
        g.close()
        g = H.HectorSlam(batch=B, max_points=nr, stream=sp, **kw)
        prof["device"] = kernel_ms(lambda: fl.device_arm(g))
        g.close()
    except Exception as e:  # the end-to-end numbers stand on their own
        prof = {"error": repr(e)}

    scans = B * n
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {
        "scans": scans, "map_updates": updates, "kept_beams_mean": round(float(fl.cnt.mean()), 1),
        "host": {"s": round(med["host"], 4), "scans_per_s": round(scans / med["host"], 1),
                 "convert_s": round(med["host_convert"], 4), "event_ms": round(med["host_event_ms"], 2),
                 "h2d_bytes": fl.h2d_host_arm(), "all_s": [round(x, 4) for x in times["host"]]},
        "device": {"s": round(med["device"], 4), "scans_per_s": round(scans / med["device"], 1),
                   "event_ms": round(med["device_event_ms"], 2), "h2d_bytes": fl.h2d_device_arm(),
                   "all_s": [round(x, 4) for x in times["device"]]},
        "device_over_host": round(med["host"] / med["device"], 3),
        "kernel_ms": prof,
        "identical": equal,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--processors", type=int, default=128)
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--worlds", default="room,hall")
    ap.add_argument("--modes", default="exact,fast")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5000)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    H, M, R = pkg.load("hector"), pkg.load("matcher"), pkg.load("rosio")
    if M.device_count() < 1:
        raise SystemExit("hector_scan_bench: no CUDA device")
    recs = {}
    for world in a.worlds.split(","):
        t0 = time.perf_counter()
        jobs = [(world, a.seed + 1000 * (world == "hall") + b, a.scans) for b in range(a.processors)]
        with ProcessPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
            rec = list(ex.map(recording, jobs))
        recs[world] = (np.stack([r[0] for r in rec]), np.stack([r[1] for r in rec]), time.perf_counter() - t0)
    import torch
    torch.cuda.init()
    result = {"workload": f"{a.processors} Hector processors x {a.scans} self-driven LaserScans each (1081 float32 "
                          "ranges), 1000 x 1000 x 3-level maps at 0.05 m, node defaults",
              "card": card(), "device": torch.cuda.get_device_name(0), "worlds": {}}
    for world, (firsts, ranges, secs) in recs.items():
        entry = {"recordings_s": round(secs, 1)}
        for mode in a.modes.split(","):
            entry[mode] = run(H, R, ranges, firsts, mode == "exact", a.repeats)
        result["worlds"][world] = entry
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
