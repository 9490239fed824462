"""Throughput of the lesson3 PL-ICP odometry node for a mixed fleet of robots (b2s_plicp_odom_create_fleet).

  python tools/plicp_odometry_fleet_bench.py [--fleets 32,132] [--scans 100] [--repeats 3]

B recordings of four robot types, recording b of type b % 4, each type with its own laser, mount and parameters:
  1081 beams over 270 deg, 720 over 360 deg, 1440 over 360 deg, 360 over 360 deg.
Recordings are synthetic drives (synth.py) from a pool of scans per type; recording b starts at pool offset b // 4.
The same recordings run three ways, each end to end (host ranges in, outputs on the host), after a warm-up:
  * fleet:  one fleet handle, every recording in one call (one launch);
  * types:  one b2s_plicp_odom_create handle per robot type, called in turn;
  * single: one handle per recording, called in turn.
The three outputs must be identical byte for byte.  Reports the best of --repeats per way, with the card's name and
power limit read in the same run.  Prints one JSON line; nothing is written to the tree."""
from __future__ import annotations

import argparse
import importlib
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
from plicp_odometry_bench import card  # noqa: E402


def robot_types():
    """(name, n_beams, angle_min, angle_increment (float32), mount, parameter overrides) of the four robot types."""
    d = math.radians

    def q_yaw(y):
        return (0.0, 0.0, math.sin(y / 2), math.cos(y / 2))

    return [
        ("1081x270", 1081, np.float32(d(-135)), np.float32(d(0.25)), (0.1, 0.0, 0.2) + q_yaw(0.0), {}),
        ("720x360", 720, np.float32(-math.pi), np.float32(2 * math.pi / 720), (0.0, 0.05, 0.3) + q_yaw(0.2),
         dict(kf_dist_linear=0.15, kf_scan_count=8)),
        ("1440x360", 1440, np.float32(-math.pi), np.float32(2 * math.pi / 1440), (-0.1, 0.0, 0.25) + q_yaw(-0.3),
         dict(kf_dist_angular=0.06, max_iterations=8)),
        ("360x360", 360, np.float32(-math.pi), np.float32(2 * math.pi / 360), (0.0, 0.0, 0.15) + q_yaw(math.pi),
         dict(kf_scan_count=5, max_correspondence_dist=0.8)),
    ]


def odom_params(abi, mount, over):
    over = dict(over)
    icp = abi.icp_params(**{k: over.pop(k) for k in list(over) if hasattr(abi.IcpParams, k)})
    return abi.plicp_odom_params(icp=icp, base_to_laser=mount, **over)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fleets", default="32,132")
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    abi, synth = pkg.abi, pkg.synth
    P = pkg.load("plicp")
    types = robot_types()
    S = a.scans
    pools, params = [], []
    for t, (_, n, amin, ainc, mount, over) in enumerate(types):
        las = synth.Laser(n_readings=n, min_angle=float(amin), angular_resolution=float(ainc))
        _, _, pool = synth.make_trajectory(11 + t, S + 40, las, step_xy=0.02, step_th_deg=0.5)
        pools.append(pool.astype(np.float32))
        params.append(odom_params(abi, mount, over))
    t = np.arange(S) * 100_000_000
    stamps = np.stack([100 + t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)
    limits = np.tile(np.float32([0.1, 30.0]), (S, 1))
    res = {"types": [ty[0] for ty in types], "scans_per_recording": S, "runs": []}

    def best(fn):
        fn()  # warm-up (allocations, module load)
        times, out = [], None
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            out = fn()
            times.append(time.perf_counter() - t0)
        return min(times), out

    for B in [int(x) for x in a.fleets.split(",")]:
        kind = [b % 4 for b in range(B)]
        recs = [pools[k][(b // 4) % 40:(b // 4) % 40 + S] for b, k in enumerate(kind)]
        beams = sum(types[k][1] for k in kind) * S
        fleet = P.Odometry.fleet([params[k] for k in kind], [types[k][1] for k in kind], [types[k][2] for k in kind],
                                 [types[k][3] for k in kind])

        def run_fleet():
            fleet.reset()
            return fleet.process(recs, [stamps] * B, [limits] * B)

        per_type = [P.Odometry(params[k], kind.count(k), types[k][1], float(types[k][2]), float(types[k][3]), 0.1, 30.0)
                    for k in range(4)]

        def run_types():
            out = [None] * B
            for k, h in enumerate(per_type):
                h.reset()
                idx = [b for b in range(B) if kind[b] == k]
                for b, o in zip(idx, h.process([recs[b] for b in idx], [stamps] * len(idx))):
                    out[b] = o
            return out

        singles = [P.Odometry.fleet([params[k]], [types[k][1]], [types[k][2]], [types[k][3]]) for k in kind]

        def run_single():
            out = []
            for b, h in enumerate(singles):
                h.reset()
                out.append(h.process([recs[b]], [stamps], [limits])[0])
            return out

        row = {"B": B, "scans": B * S, "beams": beams}
        outs = {}
        for way, fn in (("fleet", run_fleet), ("types", run_types), ("single", run_single)):
            dt, outs[way] = best(fn)
            row[way] = {"seconds": dt, "scans_per_s": B * S / dt}
        for way in ("types", "single"):
            assert all(x.tobytes() == y.tobytes() for x, y in zip(outs[way], outs["fleet"])), f"{way} differs from fleet"
        row["identical"] = True
        row["valid_fraction"] = float(np.mean(np.concatenate([o["valid"][1:] for o in outs["fleet"]])))
        res["runs"].append(row)
        for h in [fleet] + per_type + singles:
            h.close()
    res["card"], res["power_limit"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
