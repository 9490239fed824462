"""Crafted inputs for the ray-tracing tests of the Karto occupancy grid (K2c) and the GMapping map (K2b), shared by
test_raytrace_reference.py (CPU) and test_gpu_raytrace_edges.py (device).  Inputs only: every expected value comes
from raytrace_reference.py.

Most end points are kept at least HALF_CELL_MARGIN of a cell away from a rounding boundary, so that a last-ulp
difference between the device's cos / sin and the C library's cannot move a cell (DESIGN.md §4, numerics policy);
the tests assert this.  The deliberate rounding ties sit on headings 0 and pi, where both give cos exactly +-1."""
from __future__ import annotations

import ctypes
import importlib
import math
from dataclasses import dataclass

import numpy as np

import raytrace_reference as rr

abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")
synth = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.synth")

HALF_CELL_MARGIN = 1e-6
RES = 0.0625  # a power of two: grid coordinates of cell-aligned positions are exact
SHORT = [(dx, dy) for dx in range(-24, 25) for dy in range(-24, 25) if (dx, dy) != (0, 0)]
STRIDE_LENGTHS = (31, 32, 33, 63, 64, 65)
TIE_SLOPES = ((1, 2), (3, 2), (1, 4), (3, 4), (5, 2), (1, 8))  # dy/dx with exact midpoint ties in the walk


def octants(length, minors=(0, 1, 2, 3)):
    """targets of a dominant length in all eight octants, with minor components over `minors` fractions / 6"""
    out = []
    for k in minors:
        m = length * k // 6 if k else 0
        for a, b in ((length, m), (m, length)):
            for sa in (1, -1):
                for sb in (1, -1):
                    out.append((sa * a, sb * b))
    out += [(length, length), (-length, length), (length, -length), (-length, -length)]  # exact diagonals
    return sorted(set(out))


def tie_targets(scale):
    out = []
    for num, den in TIE_SLOPES:
        for sx in (1, -1):
            for sy in (1, -1):
                out += [(sx * den * scale, sy * num * scale), (sx * num * scale, sy * den * scale)]
    return out


# ------------------------------------------------------------------------------------------------------- Karto

@dataclass
class KartoCase:
    laser: abi.Laser
    ranges: np.ndarray  # [scans, n_readings]
    poses: np.ndarray   # [scans, 3] robot poses
    resolution: float
    bbox: list | None = None  # explicit grid box (the shard entry point), None = CreateFromScans' own box
    ties: np.ndarray | None = None  # [scans, n_readings] beams whose end point is a deliberate rounding tie


def laser(n=1, min_angle=0.0, ares=0.0, min_range=0.0, max_range=400.0, threshold=300.0, offset=(0.0, 0.0, 0.0)):
    return abi.Laser(n, 0, min_angle, ares, min_range, max_range, threshold, (ctypes.c_double * 3)(*offset))


def single_beam_sweep(targets, origin=(0.5, -0.25), anchor=None, res=RES):
    """One single-beam scan per target cell offset (dx, dy): the robot at a cell-aligned `origin` heading along the
    beam, range hypot * res.  Two heading-pi beams of `anchor` cells make the box's minimum x exact, and ties at
    headings 0 / pi land on exact half cells."""
    sx, sy = origin
    anchor = anchor or (max(0, max(-dx for dx, _ in targets)) + 40)  # beyond every target and tie
    poses, ranges, ties = [], [], []
    for dx, dy in targets:
        poses.append((sx, sy, math.atan2(dy, dx)))
        ranges.append(math.hypot(dx, dy) * res)
        ties.append(False)
    poses.append((sx, sy, 0.0))  # zero-length ray: the end point rounds into the sensor's cell
    ranges.append(0.25 * res)
    ties.append(False)
    poses.append((sx, sy, math.pi))
    ranges.append(anchor * res)
    ties.append(False)
    for m in (0, 1, 2, 5, 16, 31):  # x = sensor + (m + 0.5) cells at heading 0 rounds up, at heading pi towards +x
        for h in (0.0, math.pi):
            poses.append((sx, sy, h))
            ranges.append((m + 0.5) * res)
            ties.append(True)
    n = len(poses)
    return KartoCase(laser(), np.array(ranges).reshape(n, 1), np.array(poses), res, None,
                     np.array(ties).reshape(n, 1))


def karto_sweep():
    targets = SHORT + tie_targets(3) + tie_targets(7)
    for L in STRIDE_LENGTHS:
        targets += octants(L)
    return single_beam_sweep(sorted(set(targets)))


def karto_long():
    """1000- and 4000-cell rays in both dominant axes, kept in thin boxes so the grids stay small"""
    x_major = [(1000, 37), (1000, -500), (4000, 64), (4000, -129), (4000, 2000), (1000, 0)]
    y_major = [(33, -1000), (-500, -1000), (-17, -4000), (129, -4000), (-2000, -4000), (0, -1000)]
    return {"long_x": single_beam_sweep(x_major), "long_y": single_beam_sweep(y_major)}


def range_boundary_case(equal_threshold):
    """one beam per filter edge of AddScan (Karto.h:5871-5887) and of the box filter (:5382)"""
    min_r, max_r = 0.1, 8.0
    thr = max_r if equal_threshold else 6.0
    vals = [min_r, np.nextafter(min_r, np.inf), max_r, np.nextafter(max_r, -np.inf),
            thr - rr.KT_TOLERANCE, np.nextafter(thr - rr.KT_TOLERANCE, -np.inf), thr, (thr + max_r) / 2,
            np.nan, np.inf, -np.inf, -0.0, 0.0, -1.0, 3.3]
    n = len(vals)
    las = laser(n, min_angle=0.3, ares=0.37, min_range=min_r, max_range=max_r, threshold=thr)
    return KartoCase(las, np.array([vals, vals[::-1]]), np.array([[0.3, -0.2, 0.1], [-0.45, 0.6, -2.0]]), 0.05)


def room_scans(n_readings, n_scans=2, seed=3, shift=(0.0, 0.0), offset=(0.0, 0.0, 0.0), threshold=7.5):
    span = synth.deg2rad(270.0)
    ares = span / (n_readings - 1) if n_readings > 1 else synth.deg2rad(1.0)
    s = synth.Laser(n_readings=n_readings, min_angle=-span / 2, max_angle=span / 2, angular_resolution=ares,
                    min_range=0.1, max_range=30.0, range_threshold=threshold, offset_pose=offset)
    _, poses, ranges = synth.make_trajectory(seed, n_scans, s, step_xy=0.3, step_th_deg=8)
    poses = poses + np.array([shift[0], shift[1], 0.0])
    return abi.laser_from(s), ranges, poses


def karto_shapes():
    """beam counts around the warp / block sizes, resolutions 0.01 ... 1, far offsets and a mounted laser"""
    out = {}
    spec = [(1, 0.05), (31, 0.01), (32, 0.05), (33, 0.25), (255, 0.05), (256, 1.0), (257, 0.25), (4097, 0.25),
            (16384, 1.0)]
    for i, (n, res) in enumerate(spec):
        shift = ((1e4, -1e4), (-1e4, 1e4), (0.0, 0.0))[i % 3]
        offset = (0.12, -0.03, 0.05) if i % 2 else (0.0, 0.0, 0.0)
        las, ranges, poses = room_scans(n, seed=10 + i, shift=shift, offset=offset)
        out[f"n{n}_res{res}"] = KartoCase(las, ranges, poses, res)
    return out


def karto_clipped():
    """grids smaller than their rays (the shard entry point): 7 x 5, 1 x 1 and a box away from the sensor, plus
    widths with width % 8 = 0, 1 and 7, and a scan list whose readings all exceed the threshold (a 0 x 0 grid)"""
    res = 0.125
    las, ranges, poses = room_scans(361, seed=5)
    sx, sy = poses[0, 0], poses[0, 1]
    out = {
        "box7x5": KartoCase(las, ranges, poses, res, [sx - 0.33, sy - 0.21, sx - 0.33 + 7 * res, sy - 0.21 + 5 * res]),
        "box1x1": KartoCase(las, ranges, poses, res, [sx - 0.04, sy - 0.09, sx - 0.04 + res, sy - 0.09 + res]),
        "off_sensor": KartoCase(las, ranges, poses, res, [sx + 1.01, sy - 0.52, sx + 2.51, sy + 0.77]),
    }
    for w in (64, 65, 71):
        out[f"width{w}"] = KartoCase(las, ranges, poses, 0.25, [sx - 7.9, sy - 5.1, sx - 7.9 + w * 0.25,
                                                                 sy - 5.1 + 41 * 0.25])
    far = laser(9, min_angle=-1.0, ares=0.25, min_range=0.1, max_range=30.0, threshold=5.0)
    out["all_beyond_threshold"] = KartoCase(far, np.full((2, 9), 12.0), np.array([[1.0, 2.0, 0.3], [1.0, 2.0, 0.4]]),
                                            0.05)
    return out


def karto_cases():
    """every crafted Karto case: name -> KartoCase"""
    out = {"sweep": karto_sweep(), "range_lt": range_boundary_case(False), "range_eq": range_boundary_case(True)}
    out.update(karto_long())
    out.update(karto_shapes())
    out.update(karto_clipped())
    return out


def karto_end_margins(case):
    """distance of every traced end point's (and sensor's) grid coordinate from a .5 rounding boundary, except the
    deliberate ties; inf where there is nothing traced"""
    las = case.laser
    bbox = case.bbox if case.bbox is not None else rr.union_bbox(las, case.ranges, case.poses)
    scale = 1.0 / case.resolution
    worst = math.inf
    for s in range(len(case.poses)):
        (sx, sy), pts = rr.point_readings(las, case.ranges[s], case.poses[s])
        coords = [sx, sy]
        for i, (px, py) in enumerate(pts):
            r = float(case.ranges[s, i])
            if r <= las.min_range or r >= las.max_range or math.isnan(r):
                continue
            if case.ties is not None and case.ties[s, i]:
                continue
            if r >= las.range_threshold:
                ratio = las.range_threshold / r
                px, py = sx + ratio * (px - sx), sy + ratio * (py - sy)
            coords += [px, py]
        for k, v in enumerate(coords):
            g = (v - bbox[k % 2]) * scale
            worst = min(worst, abs(abs(g - math.floor(g)) - 0.5))
    return worst


THRESHOLD_PAIRS = [(0, 0), (1, 1), (2, 2), (2, 1), (3, 0), (3, 1), (3, 3), (10, 1), (100, 10), (100, 11),
                   (4294967295, 429496729), (4294967295, 429496730), (4294967295, 4294967295), (4294967295, 0),
                   (4294967294, 429496729), (2147483648, 214748365), (2147483648, 214748364), (30, 3), (31, 3),
                   (1000000, 100000), (1000000, 100001), (5, 4294967295)]


# ---------------------------------------------------------------------------------------------------- GMapping

@dataclass
class GMapCall:
    ranges: np.ndarray
    angles: np.ndarray
    laser_xy: tuple
    max_range: float = 30 - 0.01
    max_urange: float = 25.0
    ties: np.ndarray | None = None


@dataclass
class GMapCase:
    bounds: tuple  # xmin, ymin, xmax, ymax, delta
    calls: list


def gmap_beams_to(targets, delta):
    """beams from a laser on a cell centre to target cell offsets (angle atan2, range hypot * delta)"""
    ang = np.array([math.atan2(dy, dx) for dx, dy in targets])
    rng = np.array([math.hypot(dx, dy) * delta for dx, dy in targets])
    return rng, ang


def gmap_sweep():
    d = RES
    # 256 x 256 cells, centre cell 128; the centre and every cell centre sit half a cell off the world axes, so no hit
    # coordinate is 0 but for the last ulp of cos / sin (its float32 sum would keep that ulp, where the device and the
    # C library may differ).  All cell centres and half cells stay exact binary fractions.
    h = d / 2
    bounds = (-8.0 + h, -8.0 + h, 8.0 + h, 8.0 + h, d)
    calls = []
    long = []
    for L in STRIDE_LENGTHS + (95, 96, 97):
        long += octants(L)
    for cell, targets in (((0, 0), SHORT + tie_targets(5) + long), ((3, -5), SHORT), ((-40, 17), SHORT)):
        r, a = gmap_beams_to(targets, d)
        # p1 == p0: a beam shorter than half a cell (only its hit is counted)
        r, a = np.append(r, [0.25 * d, 0.3 * d]), np.append(a, [0.0, 2.0])
        calls.append(GMapCall(r, a, (h + cell[0] * d, h + cell[1] * d), ties=np.zeros(len(r), bool)))
    # half-cell ties at angles 0 and pi, on both sides of the map centre: round() goes away from zero
    for cell, beams in (((2, 0), [(0.5, 0.0), (4.5, math.pi), (9.5, math.pi)]),
                        ((-5, 3), [(2.5, 0.0), (1.5, math.pi), (7.5, 0.0), (5.5, 0.0)])):
        r = np.array([m * d for m, _ in beams])
        a = np.array([hd for _, hd in beams])
        calls.append(GMapCall(r, a, (h + cell[0] * d, h + cell[1] * d), ties=np.ones(len(r), bool)))
    return GMapCase(bounds, calls)


def gmap_range_filters():
    """ComputeMap's filters (gmapping.cc:193-197, 218): zero, -0, the max_range edge, the max_urange edge, negative,
    NaN and infinite readings, and max_urange above max_range"""
    calls = []
    for max_r, max_u in ((6.0, 5.0), (6.0, 7.0)):
        vals = [0.0, -0.0, max_r, np.nextafter(max_r, np.inf), max_u, np.nextafter(max_u, -np.inf), -1.3, np.nan,
                np.inf, -np.inf, 2.0, 5.9]
        ang = 0.37 + 0.41 * np.arange(len(vals))
        calls.append(GMapCall(np.array(vals), ang, (0.1, -0.2), max_r, max_u))
    return GMapCase((-8.0, -8.0, 8.0, 8.0, 0.05), calls)


def random_beams(case_bounds, laser_xy, n, seed, margin=1):
    """n beams towards random cells of the map storage (at least `margin` cells from its edges), each aimed within
    0.4 cell of the cell's centre"""
    d = case_bounds[4]
    ref = rr.GMapReference(*case_bounds)
    rng = np.random.default_rng(seed)
    gx = rng.integers(margin, ref.size_x - margin, n) + rng.uniform(-0.4, 0.4, n)
    gy = rng.integers(margin, ref.size_y - margin, n) + rng.uniform(-0.4, 0.4, n)
    tx, ty = ref.cx + (gx - ref.sx2) * d, ref.cy + (gy - ref.sy2) * d
    return np.hypot(tx - laser_xy[0], ty - laser_xy[1]), np.arctan2(ty - laser_xy[1], tx - laser_xy[0])


def room_beams(laser_xy, walls, n=1081):
    """a 270-degree scan of n beams inside the box walls = (x_min, y_min, x_max, y_max)"""
    ang = np.array([synth.deg2rad(-135.0) + i * synth.deg2rad(270.0) / (n - 1) for i in range(n)])
    out = []
    for a in ang:
        c, s = math.cos(a), math.sin(a)
        t = math.inf
        for dist, comp in ((walls[2] - laser_xy[0], c), (walls[0] - laser_xy[0], c), (walls[3] - laser_xy[1], s),
                           (walls[1] - laser_xy[1], s)):
            if comp != 0.0 and dist / comp > 0:
                t = min(t, dist / comp)
        out.append(t)
    return np.array(out), ang


def gmap_shapes():
    """storage (32-cell patches) against the published map: narrower, equal and one column wider, taller storage,
    odd half sizes; plus the 512 x 512 storage under a 511-wide published map with a wall in its last column"""
    out = {}
    shapes = {
        "msx_lt_width_msy_gt_height": (-3.0, -3.0, 3.25, 2.96875, RES),   # storage 96 x 96, published 100 x 95
        "odd_half_sizes": (-3.0, -2.0, 3.125, 2.125, RES),                  # storage 96 x 64, published 98 x 66
        "msx_eq_width": (-4.0, -2.0, 4.0, 2.0, RES),                         # storage 128 x 64, published 128 x 64
        "msx_eq_width_plus_1": (-2.0, -1.0, 1.96875, 1.03125, RES),         # storage 64 x 32, published 63 x 32
    }
    for k, (name, b) in enumerate(shapes.items()):
        ref = rr.GMapReference(*b)
        calls = []
        for j, lxy in enumerate(((ref.cx, ref.cy), (ref.cx - 7.3 * RES, ref.cy + 3.1 * RES))):
            r, a = random_beams(b, lxy, 400, seed=100 * k + j, margin=0)
            # beams into the last storage column and row (the cells that collide in the published map)
            last_x = ref.cx + (ref.size_x - 1 - ref.sx2) * RES
            ys = ref.cy + (np.arange(1, ref.size_y - 1, 3) - ref.sy2 + 0.2) * RES
            r = np.concatenate([r, np.hypot(last_x - lxy[0], ys - lxy[1])])
            a = np.concatenate([a, np.arctan2(ys - lxy[1], last_x - lxy[0])])
            calls.append(GMapCall(r, a, lxy))
        out[name] = GMapCase(b, calls)
    # the published map is 511 wide over 512-wide storage: cell (511, y) and cell (0, y + 1) share a byte
    r, a = room_beams((2.0, 0.0), (-1.0, -6.0, 12.74, 6.0))
    out["defect_row_wrap"] = GMapCase((-12.8, -12.8, 12.79, 12.79, 0.05), [GMapCall(r, a, (2.0, 0.0))])
    return out


def gmap_growth():
    """one handle, scans of 4097, 100 and 10000 beams (the scan buffers grow and shrink), then 300 beams onto five
    cells (several hits per cell for the float accumulators)"""
    b = (-8.0, -8.0, 8.0, 8.0, 0.05)
    calls = []
    for j, (n, lxy) in enumerate(((4097, (0.0, 0.0)), (100, (1.3, -2.2)), (10000, (-3.1, 0.7)))):
        r, a = random_beams(b, lxy, n, seed=7 + j)
        calls.append(GMapCall(r, a, lxy))
    rng = np.random.default_rng(11)
    cells = np.array([[2.0, 1.0], [-3.0, 4.5], [5.5, -5.5], [-0.35, -0.15], [6.0, 6.0]])
    pick = rng.integers(0, len(cells), 300)
    t = cells[pick] + rng.uniform(-0.02, 0.02, (300, 2))
    lxy = (0.35, 0.25)
    calls.append(GMapCall(np.hypot(t[:, 0] - lxy[0], t[:, 1] - lxy[1]), np.arctan2(t[:, 1] - lxy[1], t[:, 0] - lxy[0]),
                          lxy))
    return GMapCase(b, calls)


def gmap_cases():
    """every crafted GMapping case: name -> GMapCase"""
    out = {"sweep": gmap_sweep(), "range_filters": gmap_range_filters(), "growth": gmap_growth()}
    out.update(gmap_shapes())
    return out


def gmap_end_margin(case, call):
    """distance of every kept beam's (x - cx) / delta, (y - cy) / delta from a .5 boundary, except deliberate ties"""
    xmin, ymin, xmax, ymax, d = case.bounds
    cx, cy = (xmin + xmax) / 2.0, (ymin + ymax) / 2.0
    worst = math.inf
    lx, ly = call.laser_xy
    for i in range(len(call.ranges)):
        r = float(call.ranges[i])
        if r > call.max_range or r == 0.0 or not math.isfinite(r) or (call.ties is not None and call.ties[i]):
            continue
        r = min(r, call.max_urange)
        for v in ((lx + r * math.cos(call.angles[i]) - cx) / d, (ly + r * math.sin(call.angles[i]) - cy) / d,
                  (lx - cx) / d, (ly - cy) / d):
            worst = min(worst, abs(abs(v - math.floor(v)) - 0.5))
    return worst
