"""Crafted LaserScan calls for lesson4's make-map nodes (b2s_gmapping_node_maps, b2s_hector_mapping_node_maps), each
named for the rule of csrc/lesson4_node_maps.cu it exercises: PublishMap's wrapped rows with visited cells, every line
octant near half cells, the packed counters and the occupancy threshold at B2S_NODE_MAPS_MAX_RANGES beams, a laser cell
outside the storage, Hector's beam-order rule on crossing beams, its shortest beams and map edges, and maps large
enough that every chunk holds one scan.  Shared by the CPU test against the unmodified nodes and the C restatement and
by the GPU test."""
from __future__ import annotations

import importlib
import math

import numpy as np

from raytrace_reference import gmap_layout
import node_maps_reference as nr

node_maps = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.node_maps")
GP, HP = node_maps.gmapping_params, node_maps.hector_params

F32 = np.float32
FULL = 16384  # B2S_NODE_MAPS_MAX_RANGES


def fields(amin, inc, range_min=0.1, range_max=30.0):
    return F32(amin), F32(inc), F32(range_min), F32(range_max)


def circle(n, range_min=0.1, range_max=30.0):
    """n beams over a full turn from -pi"""
    return fields(-np.pi, 2 * np.pi / n, range_min, range_max)


def float_steps(v, k):
    """v moved by k float32 steps"""
    v = F32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, F32(np.inf if k > 0 else -np.inf))
    return v


def _to_walls(angles, lo, hi):
    """float32 ranges from the origin to the walls of the box [lo.x, hi.x] x [lo.y, hi.y] along `angles`"""
    c, s = np.cos(angles), np.sin(angles)
    with np.errstate(divide="ignore"):
        tx = np.where(c > 0, hi[0] / c, np.where(c < 0, lo[0] / c, np.inf))
        ty = np.where(s > 0, hi[1] / s, np.where(s < 0, lo[1] / s, np.inf))
    return np.minimum(tx, ty).astype(F32)


def _room(f, n, half, seed, scans, sigma=0.01):
    """`scans` noisy scans of the box [-half, half] around the laser"""
    rng = np.random.default_rng(seed)
    a = np.array(nr.gmapping_angles(f, n))
    return np.stack([_to_walls(a, (-half[0], -half[1]), half) + rng.normal(0, sigma, n).astype(F32)
                     for _ in range(scans)]).astype(F32)


# ------------------------------------------------------------------------------------------------------- GMapping


def storage_walls(params, n=4096):
    """One scan of n beams over a full turn whose walls run through the centres of the storage's edge cells: beams end
    in storage column msx - 1 and row msy - 1 and in column and row 0, those near the corners cross them."""
    cx, cy, msx, msy, sx2, sy2 = gmap_layout(params.xmin, params.ymin, params.xmax, params.ymax, params.delta)
    d = params.delta
    lo = ((0 - sx2) * d + cx, (0 - sy2) * d + cy)
    hi = ((msx - 1 - sx2) * d + cx, (msy - 1 - sy2) * d + cy)
    f = circle(n)
    return f, _to_walls(np.array(nr.gmapping_angles(f, n)), lo, hi)[None]


def _octant_ranges(f, n, laps):
    """ranges for a laser of bearings near k * 45 degrees: lap l of beams gives every bearing the range laps[l](c, s)"""
    a = nr.gmapping_angles(f, n)
    return np.array([[laps[i // 8](math.cos(a[i]), math.sin(a[i])) for i in range(n)]], F32)


def octant_laps(delta=0.05):
    """Per lap of 8 bearings: a range ending in the laser cell, one cell away, float neighbours of a half-cell end
    point on the dominant axis (k + 1/2 cells), past max_use_range and on it."""
    laps = [lambda c, s: F32(0.01), lambda c, s: F32(delta)]
    for k in (0, 3, 17, 160):
        for step in (-2, -1, 0, 1, 2):
            laps.append(lambda c, s, k=k, step=step: float_steps((k + 0.5) * delta / max(abs(c), abs(s)), step))
    laps += [lambda c, s: F32(27.0), lambda c, s: F32(25.0), lambda c, s: float_steps(25.0, -1)]
    return laps


def gmapping_cases():
    """name -> (params, fields, ranges [S][n])"""
    cases = {}
    # W = msx - 1: payload 511 wide, storage 512.  The laser sits 15 columns from the storage's last column, so beams
    # to the right wall cross column 511 steeply; with the laser also near the top, flat beams cross the last row.
    for name, p in (("wrap_right_edge", GP(xmin=-24.8, xmax=0.8, ymin=-12.8, ymax=12.8)),
                    ("wrap_corner", GP(xmin=-24.8, xmax=0.8, ymin=-24.8, ymax=0.8)),
                    # W = msx (1280 at 0.0625) and W > msx (999 against 992), the laser near the right edge too
                    ("exact_storage", GP(xmin=-79.0, xmax=1.0, ymin=-40.0, ymax=40.0, delta=0.0625, max_range=100.0,
                                         max_use_range=60.0)),
                    ("small_storage", GP(xmin=-49.0, xmax=1.0, ymin=-25.0, ymax=25.0, max_range=60.0,
                                         max_use_range=40.0))):
        cases[name] = (p,) + storage_walls(p)
    # bearings k * 45 degrees for k = 0 .. 191 (float sums, so each lap's bearings are float neighbours of the last's)
    f = fields(0.0, np.pi / 4)
    laps = octant_laps()
    cases["octants"] = (GP(), f, _octant_ranges(f, 8 * len(laps), laps))
    # the laser cell's boundary 5 mm to its +x side and max_use_range 2 cm: end cells on the laser cell and one cell
    # away, with and without a hit
    ll = [lambda c, s: F32(0.004), lambda c, s: F32(0.01), lambda c, s: F32(0.019), lambda c, s: F32(0.02),
          lambda c, s: F32(0.03), lambda c, s: F32(1.0)]
    cases["laser_cell_lines"] = (GP(xmin=-40.02, xmax=39.98, max_use_range=0.02), f, _octant_ranges(f, 8 * len(ll), ll))
    # B2S_NODE_MAPS_MAX_RANGES beams: n and visits of the laser cell at 16384, and at n / visits = 0.25 exactly
    f = circle(FULL)
    tiny, long_ = F32(0.01), F32(1.0)
    cases["laser_cell_all"] = (GP(), f, np.full((1, FULL), tiny, F32))
    for name, k in (("thresh_equal", 4096), ("thresh_over", 4097)):
        r = np.full(FULL, long_, F32)
        r[::4] = tiny
        if k > 4096:
            r[1] = tiny
        cases[name] = (GP(), f, r[None].copy())
    # the laser's cell (-10, 800) lies left of the storage: a scan with no kept beam is mapped, the next is refused
    f = circle(64)
    r = np.full((3, 64), F32(5.0), F32)
    r[0] = np.tile(np.array([np.nan, 0.0, np.inf, 35.0], F32), 16)
    r[1] = np.nan
    r[1, 32] = 5.0  # bearing 0: its end cell (90, 800) lies inside
    cases["laser_outside"] = (GP(xmin=0.5, xmax=40.0), f, r)
    # 8192^2 counters (256 MiB) plus a 8191^2 payload per scan: one scan per chunk
    cases["one_scan_chunks"] = (GP(xmin=-204.8, ymin=-204.8, xmax=204.8, ymax=204.8), f,
                                _room(f, 64, (12.0, 7.0), 3, 3))
    return cases


# --------------------------------------------------------------------------------------------------------- Hector


def _hector_ranges(f, n, laps, per_lap=8):
    """ranges for a laser of bearings accumulated as the node does: lap l gives bearing i the range laps[l](c, s)"""
    angle, out = F32(f[0]), []
    for i in range(n):
        c, s = math.cos(float(angle)), math.sin(float(angle))
        out.append(laps[i // per_lap](c, s))
        angle = F32(angle + f[1])
    return np.array([out], F32)


def _cells_away(m):
    """a range whose point lies m cells (of 0.05 m) from the begin cell on its dominant axis"""
    return lambda c, s: F32(m * 0.05 / max(abs(c), abs(s)))


def _boundary(m, step):
    """float neighbours of the range whose dominant coordinate is m cells exactly (a rounding boundary of p / 0.05 for
    half-integer m)"""
    return lambda c, s: float_steps(m * 0.05 / max(abs(c), abs(s)), step)


def hector_cases():
    """name -> (params, fields, ranges [S][n])"""
    cases = {}
    # adjacent bearings 0.25 degrees apart alternate short and long: a long beam's line runs over the end cells of the
    # short beams on either side, one earlier and one later in beam order
    n = 1440
    f = circle(n)
    i = np.arange(n)
    r = np.where(i % 2 == 0, 1.0 + 0.5 * ((i // 2) % 5), 6.0 + (i // 2) % 3).astype(F32)
    cases["comb"] = (HP(), f, r[None].copy())
    # range_min lowered: end cells on the begin cell (not drawn), one cell away (only the begin cell freed), and the
    # float neighbours of the +-1/2 and +-3/2 cell rounding boundaries, on every octant's bearing
    f = fields(0.0, np.pi / 4, range_min=1e-4)
    laps = [lambda c, s: F32(0.001), _cells_away(1)]
    for m in (0.5, 1.5):
        laps += [_boundary(m, k) for k in (-2, -1, 0, 1, 2)]
    cases["short_beams"] = (HP(), f, _hector_ranges(f, 8 * len(laps), laps))
    # end cells on the map's first and last rows and columns (drawn), one beyond (dropped), and the float neighbours
    # of the rounding boundary between them
    f = fields(0.0, np.pi / 4, range_max=100.0)
    laps = []
    for edge in (798, 800):  # the last column / row is 800 + 798, the first 800 - 800
        laps += [_cells_away(edge), _cells_away(edge + 1)] + [_boundary(edge + 0.5, k) for k in (-1, 0, 1)]
    cases["map_edges"] = (HP(), f, _hector_ranges(f, 8 * len(laps), laps))
    # the begin cell (800, 800) on a map's last column, and one column outside it
    room = _room(circle(720), 720, (6.0, 4.0), 7, 1)
    cases["begin_last_column"] = (HP(xmin=-20.03, xmax=20.03), circle(720), room)
    cases["begin_outside"] = (HP(xmin=-20.005, xmax=20.005), circle(720), room)
    # a 0.04 m map: end cells still step 0.05 m (updateByScanJustOnce's constant)
    cases["delta_004"] = (HP(delta=0.04), circle(720), _room(circle(720), 720, (30.0, 20.0), 8, 2))
    # a 16399^2 payload (256.5 MiB): one scan per chunk
    f = circle(64)
    cases["one_scan_chunks"] = (HP(xmin=-410.0, ymin=-410.0, xmax=410.0, ymax=410.0), f, _room(f, 64, (12.0, 7.0), 9, 3))
    return cases

