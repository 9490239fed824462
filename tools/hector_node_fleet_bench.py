"""Time a mixed fleet of lesson4 Hector SLAM nodes in one handle (b2s_hector_node_create_fleet) against the two ways the
same robots ran before it: one b2s_hector_node_create_batch handle per robot type, called one after another, and one
single-node handle per robot, called one after another.  Each robot type has its own laser and map:

  hokuyo    1081 beams, 270 deg, 0.1-30 m    2048 x 2048 at 0.05 m, 3 levels (the node's defaults)
  lidar720   720 beams, 360 deg, 0.12-16 m   1024 x 1024 at 0.05 m, 3 levels
  dense1440 1440 beams, 360 deg, 0.2-25 m    2048 x 2048 at 0.025 m, 4 levels
  small360   360 beams, 360 deg, 0.15-12 m    512 x  512 at 0.1 m, 2 levels

Node b is of type b mod 4 and replays a seeded synthetic walk (synth.make_trajectory with its type's laser) at 40 Hz,
starting at its own place in the walk.  Host ranges in, maps handed to a callback on the host.

  python tools/hector_node_fleet_bench.py [--scans 400] [--batch 32] [--period 1e6] [--repeat 3]

The three ways must give identical outputs: poses, covariances, gate flags, kept-beam counts, the maps handed out
(CRC-32 of each payload with its stamp and scan index) and every node's final map (publish_map after the timed call).
The tool fails if they do not.  Prints one JSON line: per way the best and median seconds over --repeat runs and
scans/s, and the card's name and power limit, read in the same run.  It needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
from hector_node_bench import card  # noqa: E402

# name: (beams, field of view deg, range_min, range_max, map_size, map_resolution, levels)
TYPES = {"hokuyo": (1081, 270.0, 0.1, 30.0, 2048, 0.05, 3), "lidar720": (720, 360.0, 0.12, 16.0, 1024, 0.05, 3),
         "dense1440": (1440, 360.0, 0.2, 25.0, 2048, 0.025, 4), "small360": (360, 360.0, 0.15, 12.0, 512, 0.1, 2)}
NAMES = list(TYPES)


def laser_of(name):
    beams, fov = TYPES[name][:2]
    inc = np.deg2rad(fov) / (beams if fov == 360.0 else beams - 1)
    amin = -np.deg2rad(fov) / 2
    return pkg.synth.Laser(n_readings=beams, min_angle=amin, max_angle=amin + inc * (beams - 1), angular_resolution=inc,
                           min_range=TYPES[name][2], max_range=TYPES[name][3])


def geometry_of(R, name):
    las = laser_of(name)
    amin, inc = np.float32(las.min_angle), np.float32(las.angular_resolution)
    return R.make_msg(amin, amin + inc * np.float32(las.n_readings - 1), inc, np.float32(las.min_range),
                      np.float32(las.max_range), np.zeros(las.n_readings, np.float32))


def params_of(N, name, period):
    size, res, levels = TYPES[name][4:]
    return N.node_params(dict(map_size=size, map_resolution=res, map_multi_res_levels=levels, map_pub_period=period))


def recordings(B, n):
    """node b: type b mod 4, a 300-scan walk of its type looped forwards and backwards from scan 37 b, 40 Hz stamps"""
    loops = {}
    for k, name in enumerate(NAMES):
        _, _, base = pkg.synth.make_trajectory(20 + k, 300, laser_of(name), step_xy=0.02, step_th_deg=0.5)
        loops[name] = np.concatenate([base, base[::-1]]).astype(np.float32)
    out = []
    for b in range(B):
        loop = loops[NAMES[b % len(NAMES)]]
        idx = (37 * b + np.arange(n)) % len(loop)
        t = (1_000 + b) * 1_000_000_000 + np.arange(n, dtype=np.int64) * 25_000_000
        out.append((np.ascontiguousarray(loop[idx]), np.stack([t // 1_000_000_000, t % 1_000_000_000], 1).astype(np.uint32)))
    return out


def _collect(maps):
    def on_map(b, m):
        maps[b].append((m["scan_index"], m["stamp"], zlib.crc32(m["payload"].tobytes())))
    return on_map


def _final(h, b):
    m = h.publish_map(b, (0, 0)) if isinstance(h, pkg.load("hector_node").HectorNodeBatch) else h.publish_map((0, 0))
    return zlib.crc32(m["payload"].tobytes())


def run_fleet(N, R, recs, period):
    B = len(recs)
    h = N.HectorNodeBatch.fleet([params_of(N, NAMES[b % 4], period) for b in range(B)],
                                [geometry_of(R, NAMES[b % 4]) for b in range(B)], [(0, 0, 0, 0, 0, 0, 1)] * B)
    maps = [[] for _ in range(B)]
    t0 = time.perf_counter()
    out = h.process([r for r, _ in recs], [s for _, s in recs], on_map=_collect(maps))
    s = time.perf_counter() - t0
    final = [_final(h, b) for b in range(B)]
    h.close()
    return s, out, maps, final


def run_per_type(N, R, recs, period):
    B = len(recs)
    out, maps, final = [None] * B, [[] for _ in range(B)], [None] * B
    s = 0.0
    for k, name in enumerate(NAMES):
        nodes = list(range(k, B, len(NAMES)))
        if not nodes:
            continue
        h = N.HectorNodeBatch([params_of(N, name, period)] * len(nodes), geometry_of(R, name),
                              [(0, 0, 0, 0, 0, 0, 1)] * len(nodes))
        sub = [[] for _ in nodes]
        t0 = time.perf_counter()
        got = h.process([recs[b][0] for b in nodes], [recs[b][1] for b in nodes], on_map=_collect(sub))
        s += time.perf_counter() - t0
        for j, b in enumerate(nodes):
            out[b], maps[b], final[b] = got[j], sub[j], _final(h, j)
        h.close()
    return s, out, maps, final


def run_singles(N, R, recs, period):
    out, maps, final = [], [], []
    s = 0.0
    for b, (r, st) in enumerate(recs):
        name = NAMES[b % 4]
        node = N.HectorNode(params_of(N, name, period), geometry_of(R, name))
        mine = [[]]
        t0 = time.perf_counter()
        got = node.process(r, st, on_map=lambda m: _collect(mine)(0, m))
        s += time.perf_counter() - t0
        out.append(got), maps.append(mine[0]), final.append(_final(node, 0))
        node.close()
    return s, out, maps, final


def same(a, b):
    """two runs' outputs, bit for bit"""
    _, oa, ma, fa = a
    _, ob, mb, fb = b
    for x, y in zip(oa, ob):
        for key in ("pose", "pose_msg", "cov", "map_updated", "n_points"):
            u, v = np.asarray(x[key]), np.asarray(y[key])
            if u.shape != v.shape or not np.array_equal(u.view(np.uint8), v.view(np.uint8)):
                return False
    return ma == mb and fa == fb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=400)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--period", type=float, default=1e6)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    M = pkg.load("matcher")
    if M.device_count() < 1:
        raise SystemExit("hector_node_fleet_bench: no CUDA device (there is no CPU fallback)")
    N, R = pkg.load("hector_node"), pkg.load("rosio")
    recs = recordings(a.batch, a.scans)
    run_fleet(N, R, [(r[:50], s[:50]) for r, s in recs[:8]], 2.0)  # warm-up: module load, pools, pinned buffers
    ways = {"fleet": run_fleet, "per_type_batches": run_per_type, "single_nodes": run_singles}
    times = {k: [] for k in ways}
    first = {}
    for _ in range(a.repeat):
        for k, fn in ways.items():  # alternated, so that drift on a shared host hits every way alike
            res = fn(N, R, recs, a.period)
            times[k].append(res[0])
            first.setdefault(k, res)
    identical = same(first["fleet"], first["per_type_batches"]) and same(first["fleet"], first["single_nodes"])
    total = a.batch * a.scans
    rows = {k: dict(best_s=round(min(v), 4), median_s=round(statistics.median(v), 4),
                    scans_per_s=round(total / min(v)), runs_s=[round(x, 4) for x in v]) for k, v in times.items()}
    print(json.dumps(dict(nodes=a.batch, scans_per_node=a.scans, map_pub_period=a.period,
                          types={n: dict(zip(("beams", "fov_deg", "range_min", "range_max", "map_size", "resolution",
                                              "levels"), TYPES[n])) for n in NAMES},
                          ways=rows, identical=identical,
                          fleet_vs_per_type=round(min(times["per_type_batches"]) / min(times["fleet"]), 3),
                          fleet_vs_singles=round(min(times["single_nodes"]) / min(times["fleet"]), 3), card=card())))
    if not identical:
        raise SystemExit("hector_node_fleet_bench: the three ways disagree")


if __name__ == "__main__":
    main()
