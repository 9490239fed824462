"""Inputs for the Hector processor's edge tests (tests/test_hector_edges_reference.py, tests/test_gpu_hector_edges.py):
map geometries and scan streams, seeded, CPU only.  The file name keeps pytest from collecting it; tests import it.

Points are level-0 map-cell units in the laser frame, as `hector.scan_to_data_container` builds them; poses are float32
world poses.  A Stream is run in one of three forms (`run_stream`): "self" (hint = the previous scan-match pose, the
node's loop, starting from `first`), "hints" (one hint per scan) and "given" (`map_without_matching` at the hints).

Geometries: non-square maps both ways (one with odd halvings), a robot 2-3 m from two edges of the map, eight levels,
one level, and the smallest map a 3-level processor accepts.  Families:
- walk:   a self-driven trajectory; hints wrapped by +-2pi and +-4pi (normalize_angle's fmod branch)
- empty:  the walk with 0-point scans in the middle
- long:   4096-beam scans cut to 1 ... 2048 points (the single handle's capacity)
- batch_long: 2049 ... 4096 points (a batched handle's capacity); not for the single handle
- stamps: crafted rays on column 0, row 0, the last column and row and around rays that leave the map: several beams
          ending on one cell, lower / higher beams freeing it, zero-length rays.  Applied with map_without_matching only
- interp_edge: match points exactly on x = sx - 2 / y = sy - 2 and 2^-6 beyond (exact on the first iteration of a
          one-level map, where the first evaluation is at the hint)"""
from __future__ import annotations

import importlib
import os
import sys
from dataclasses import dataclass

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
PKG = "creating-2d-laser-slam-from-scratch_b200"
synth = importlib.import_module(PKG + ".synth")
scan_to_data_container = importlib.import_module(PKG + ".hector").scan_to_data_container

GEOMETRIES = {
    "wide": dict(size_x=640, size_y=360, resolution=0.05, start=(0.5, 0.5), levels=3),
    "tall_odd": dict(size_x=333, size_y=901, resolution=0.05, start=(0.3, 0.6), levels=4),  # 333/166/83/41 x 901/450/225/112
    "edge": dict(size_x=400, size_y=300, resolution=0.05, start=(0.15, 0.85), levels=3),
    "deep": dict(size_x=1024, size_y=768, resolution=0.025, start=(0.5, 0.5), levels=8),  # coarsest 8 x 6
    "flat": dict(size_x=512, size_y=512, resolution=0.05, start=(0.5, 0.5), levels=1),
    "tiny": dict(size_x=12, size_y=12, resolution=0.05, start=(0.5, 0.5), levels=3),  # 12 >> 2 = 3 > 2: the smallest
}
GATE = dict(min_dist=0.1, min_angle=0.9)  # the walk moves ~0.05 m a scan: the gate opens every few scans, not always
FAMILIES = ("walk", "empty", "long", "batch_long", "stamps", "interp_edge")
FORMS = {"walk": ("self", "hints", "given"), "empty": ("self", "hints", "given"), "long": ("hints", "given"),
         "batch_long": ("hints", "given"), "stamps": ("given",), "interp_edge": ("self", "hints", "given")}
SINGLE_LENGTHS = (1, 2, 3, 4, 5, 7, 8, 9, 31, 32, 33, 575, 576, 577, 1151, 1152, 1153, 2047, 2048)
BATCH_LENGTHS = (2049, 3000, 4095, 4096)
LONG_LASER = synth.Laser(n_readings=4096, angular_resolution=synth.deg2rad(270) / 4095)


@dataclass
class Stream:
    scans: list          # [n_i, 2] float32
    hints: np.ndarray    # [n, 3] float32
    first: np.ndarray    # [3] float32

    def __len__(self):
        return len(self.scans)


def processor_kw(geometry):
    return dict(GEOMETRIES[geometry], **GATE)


def _wrapped(poses):
    """float32 poses with headings moved by 0, +2pi, -2pi, +4pi, -4pi in turn (same direction, outside +-pi)."""
    h = np.asarray(poses, np.float64).copy()
    h[:, 2] += 2 * np.pi * np.array([0, 1, -1, 2, -2])[np.arange(len(h)) % 5]
    return h.astype(np.float32)


def _walk(geometry, seed, n):
    res = GEOMETRIES[geometry]["resolution"]
    laser = synth.Laser()
    _, poses, ranges = synth.make_trajectory(seed, n, laser, step_xy=0.1, step_th_deg=3)
    scans = [scan_to_data_container(ranges[i], laser, res) for i in range(n)]
    return Stream(scans, _wrapped(poses), poses[0].astype(np.float32))


def _long(geometry, seed, lengths):
    res = GEOMETRIES[geometry]["resolution"]
    _, poses, ranges = synth.make_trajectory(seed, len(lengths), LONG_LASER, step_xy=0.1, step_th_deg=3)
    scans = []
    for i, n in enumerate(lengths):
        pts = scan_to_data_container(ranges[i], LONG_LASER, res)
        assert len(pts) >= n, (len(pts), n)  # the room is closed and the robot stays in its box-free middle
        scans.append(np.ascontiguousarray(pts[:n]))
    return Stream(scans, _wrapped(poses), poses[0].astype(np.float32))


def _map_tf(geometry):
    """map_coords_pose's float32 numbers at level 0 (GridMapBase.h:238-242 with the MapRepMultiMap offset)."""
    g = GEOMETRIES[geometry]
    f = np.float32
    res = f(g["resolution"])
    lin = f(1) / res
    tx = lin * (f(res * f(g["size_x"])) * f(g["start"][0]))
    ty = lin * (f(res * f(g["size_y"])) * f(g["start"][1]))
    return lin, tx, ty


def _world_of(geometry, mx, my):
    """A heading-0 world pose whose level-0 map coordinates are within float rounding of (mx, my)."""
    lin, tx, ty = _map_tf(geometry)
    return np.array([(mx - float(tx)) / float(lin), (my - float(ty)) / float(lin), 0.0], np.float32)


def _map_of(geometry, w):
    lin, tx, ty = _map_tf(geometry)
    f = np.float32
    return (lin * f(w[0]) + f(0) * f(w[1])) + tx, (f(0) * f(w[0]) + lin * f(w[1])) + ty


def stamp_cases(geometry):
    """(robot cell, [end cells in beam order]) of the crafted stamp-order scans.  Cell k is map coordinate k (begin and
    end cells round by +0.5, OccGridMapBase.h:137-160)."""
    sx, sy = GEOMETRIES[geometry]["size_x"], GEOMETRIES[geometry]["size_y"]
    out = []
    # a robot in each corner, rays along an edge: column 0, row 0, the last column, the last row
    for r, u in (((0, 0), (0, 1)), ((sx - 1, 0), (-1, 0)), ((sx - 1, sy - 1), (0, -1)), ((0, sy - 1), (1, 0))):
        a = (r[0] + 4 * u[0], r[1] + 4 * u[1])   # the contested cell
        b = (r[0] + 6 * u[0], r[1] + 6 * u[1])   # beyond it: a ray ending here passes through a
        out += [(r, [a, b]),        # a lower beam ends on a, a higher one passes: a stays occupied, gets no free update
                (r, [b, a]),        # a lower beam frees a, a higher one ends on it: "(v + f) - f"
                (r, [a, a, a, b]),  # three beams end on a, a fourth crosses it
                (r, [b, a, a, a]),
                (r, [r, r, a])]     # zero-length rays
    # rays that leave the map are dropped whole: a cell they cross gets only what the other beams give it
    for r, u in (((3, sy // 2), (-1, 0)), ((sx // 2, 3), (0, -1)), ((sx - 4, sy // 2), (1, 0)), ((sx // 2, sy - 4), (0, 1))):
        a = (r[0] + 2 * u[0], r[1] + 2 * u[1])
        o = (r[0] + 6 * u[0], r[1] + 6 * u[1])   # outside the map
        out += [(r, [o, a]), (r, [a, o]), (r, [o, o, a, a])]
    return out


def _stamps(geometry):
    scans, hints = [], []
    for r, ends in stamp_cases(geometry):
        w = _world_of(geometry, *r)
        mx, my = _map_of(geometry, w)
        scans.append(np.array([(e[0] - float(mx), e[1] - float(my)) for e in ends], np.float32))
        hints.append(w)
    return Stream(scans, np.stack(hints), hints[0])


def _interp_edge(geometry):
    """Six scans from one heading-0 pose near the top right corner: walls on x = sx - 2 and y = sy - 2, points 2^-6
    beyond them and two inner walls that keep the Hessian regular."""
    sx, sy = GEOMETRIES[geometry]["size_x"], GEOMETRIES[geometry]["size_y"]
    d = min(10, (min(sx, sy) - 2) // 2)
    w = _world_of(geometry, sx - 2 - d, sy - 2 - d)
    mx, my = _map_of(geometry, w)
    f = np.float32
    lim_x, lim_y, eps = f(sx - 2), f(sy - 2), f(2.0 ** -6)
    t = np.linspace(-d, d - 1, 2 * d).astype(np.float32)
    pts = [np.stack([np.full_like(t, lim_x - mx), t], 1),            # exactly on x = sx - 2 (first evaluation)
           np.stack([np.full_like(t, (lim_x + eps) - mx), t + f(0.5)], 1),  # just beyond it
           np.stack([t, np.full_like(t, lim_y - my)], 1),
           np.stack([t + f(0.5), np.full_like(t, (lim_y + eps) - my)], 1),
           np.stack([np.full_like(t, f(-d) + f(0.25)), t], 1),       # inner walls
           np.stack([t, np.full_like(t, f(-d) + f(0.25))], 1)]
    p = np.ascontiguousarray(np.concatenate(pts).astype(np.float32))
    return Stream([p] * 6, np.stack([w] * 6), w)


def interp_edge_exact(geometry):
    """Whether the first evaluation of the interp_edge scan (at the hint, heading 0) lands exactly on sx - 2 and on
    sx - 2 + 2^-6."""
    sx = GEOMETRIES[geometry]["size_x"]
    s = _interp_edge(geometry)
    mx, _ = _map_of(geometry, s.hints[0])
    n = len(s.scans[0]) // 6
    x = s.scans[0][:, 0]
    return bool(((x[:n] + mx) == np.float32(sx - 2)).all() and
                ((x[n:2 * n] + mx) == np.float32(sx - 2) + np.float32(2.0 ** -6)).all())


def make_stream(geometry, family, n=14):
    seed = 100 + sorted(GEOMETRIES).index(geometry)
    if family == "walk":
        return _walk(geometry, seed, n)
    if family == "empty":
        s = _walk(geometry, seed, n)
        for i in (2, 3, 7, n - 2):
            s.scans[i] = np.zeros((0, 2), np.float32)
        return s
    if family == "long":
        return _long(geometry, seed, SINGLE_LENGTHS)
    if family == "batch_long":
        return _long(geometry, seed, BATCH_LENGTHS)
    if family == "stamps":
        return _stamps(geometry)
    if family == "interp_edge":
        return _interp_edge(geometry)
    raise KeyError(family)


def run_stream(proc, stream, form, origo=(0.0, 0.0)):
    """update() once per scan in one of the three forms.  Returns poses [n, 3] and covariances [n, 3, 3] (float32; the
    covariance is zero where nothing was matched) and, where `proc` reports it, the gate decisions [n]."""
    est = stream.first
    poses, covs, flags = [], [], []
    for i, pts in enumerate(stream.scans):
        hint = est if form == "self" else stream.hints[i]
        est, cov = proc.update(pts, origo, hint, form == "given")
        poses.append(np.asarray(est, np.float32))
        covs.append(np.zeros((3, 3), np.float32) if form == "given" else np.asarray(cov, np.float32).reshape(3, 3))
        flag = getattr(proc, "map_updated", None)  # (a recorded reference answers only through its method calls)
        if isinstance(flag, bool):
            flags.append(flag)
    return np.stack(poses), np.stack(covs), np.array(flags, bool)


def same_bits(a, b):
    """float32 arrays equal bit for bit, except that a NaN matches any NaN (x86 and the GPU write different NaN
    payloads; where a 1-3-point scan meets a singular Hessian both must produce NaN in the same places)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a.view(np.int32)[~na], b.view(np.int32)[~nb])


def cell_mismatch(a, b):
    """Cells whose log-odds bits or update index differ, over the whole plane (touched or not)."""
    (la, ua), (lb, ub) = a, b
    return int(((ua != ub) | (la.view(np.int32) != lb.view(np.int32))).sum()), int(((ua >= 0) | (ub >= 0)).sum())
