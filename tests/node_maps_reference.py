"""Brute-force builds of lesson4's make-map nodes, one scan at a time, written from the nodes' own code paths:
lesson4/src/gmapping/gmapping.cc (InitParams, CreateCache, ComputeMap, PublishMap) and
lesson4/src/hector_mapping/hector_mapping.cc with include/lesson4/hector_mapping/map/{OccGridMapBase.h,
GridMapLogOdds.h} (InitParams, ROSLaserScanToDataContainer, updateByScanJustOnce, PublishMap).

Plain Python and numpy.  The GMapping line walk, map layout and C rounding are raytrace_reference's; nothing here calls
library code, the C restatement or the closed-form lines of the kernels.  GMapping keeps separate integer n and visits
per storage cell; Hector applies its beams in order with the update-index marks and float32 log-odds, so a device that
relies on set semantics instead has to agree with it.  Cells are kept sparsely (dicts) and PublishMap runs a block of
`width` storage columns per numpy step, so maps of 8192^2 and 16384^2 cells take seconds."""
from __future__ import annotations

import math

import numpy as np

from raytrace_reference import c_round, gmap_layout, grid_line


def node_dim(d: float) -> int:
    """The nodes' conversion of a double map dimension into their unsigned / int fields (truncation)."""
    if not (1.0 <= d < 2147483648.0):
        raise ValueError(f"a map dimension of {d} cells")
    return int(d)


# ------------------------------------------------------------------------------------------------------- GMapping


def gmapping_dims(params):
    """InitParams (gmapping.cc:69-73): width / height = (max - min) / map_.info.resolution, a float32."""
    res = float(np.float32(params.delta))
    return node_dim((params.xmax - params.xmin) / res), node_dim((params.ymax - params.ymin) / res)


def gmapping_angles(fields, n):
    """CreateCache (gmapping.cc:118-123): angle_min + i * angle_increment with i unsigned, so a float product and a
    float sum, widened to double."""
    amin, inc = np.float32(fields[0]), np.float32(fields[1])
    return [float(np.float32(amin + np.float32(i) * inc)) for i in range(n)]


class GMappingScan:
    """ComputeMap (gmapping.cc:171-242) of one scan into a fresh ScanMatcherMap: n and visits per storage cell, keyed
    by (x, y).  `refused` is set where the node asserts (a kept beam whose laser cell or end cell is outside the
    storage, map.h:186-191)."""

    def __init__(self, params, angles, ranges):
        p = params
        self.cx, self.cy, self.msx, self.msy, self.sx2, self.sy2 = gmap_layout(p.xmin, p.ymin, p.xmax, p.ymax, p.delta)
        self.delta = p.delta
        self.n, self.visits = {}, {}
        self.ends, self.lines = [], []  # per kept beam: end cell, hit?; the whole p0 -> p1 list
        self.refused = False
        p0 = self.world2map(0.0, 0.0)  # lp = (0, 0, 0)
        self.p0 = p0
        hits = []
        for i in range(len(ranges)):
            d = float(ranges[i])
            if d > p.max_range or d == 0.0 or not math.isfinite(d):  # :190-191
                continue
            if d > p.max_use_range:
                d = p.max_use_range
            hx = 0.0 + d * math.cos(angles[i])
            hy = 0.0 + d * math.sin(angles[i])
            p1 = self.world2map(hx, hy)
            if not (self.inside(p0) and self.inside(p1)):
                self.refused = True
                return
            line = grid_line(p0, p1)
            assert line[0] == p0 and line[-1] == p1
            self.lines.append(line)
            self.ends.append((p1, d < p.max_use_range))
            if d < p.max_use_range:  # :214-219
                hits.append(p1)  # world2map(hit) is p1
        for line in self.lines:  # every cell but the last is free (:227-235)
            for c in line[:-1]:
                self.visits[c] = self.visits.get(c, 0) + 1
        for c in hits:  # PointAccumulator::update(true, hit): n++, visits++ (:237-241)
            self.n[c] = self.n.get(c, 0) + 1
            self.visits[c] = self.visits.get(c, 0) + 1

    def world2map(self, x, y):  # map.h:171-174
        return (int(c_round((x - self.cx) / self.delta)) + self.sx2,
                int(c_round((y - self.cy) / self.delta)) + self.sy2)

    def inside(self, c):
        return 0 <= c[0] < self.msx and 0 <= c[1] < self.msy

    def classes(self, occ_thresh):
        """gmapping_map_.cell(p) as PublishMap reads it, for every storage cell [msy][msx]: -1 unknown (no visit),
        100 where n * 1 / visits > occ_thresh (strictly), else 0."""
        out = np.full((self.msy, self.msx), -1, np.int8)
        for (x, y), v in self.visits.items():
            occ = float(self.n.get((x, y), 0)) * 1 / float(v)  # PointAccumulator::operator double (map.h:27)
            out[y, x] = 100 if occ > occ_thresh else 0
        return out


def _column_blocks(msx, msy, width, height):
    """PublishMap's x-outer loop in blocks of `width` storage columns: cells (x, y) and (x', y') share the byte
    width * y + x only when x' - x is a multiple of width, so no two cells of a block write the same byte and the
    blocks, taken in x order, write in the loop's order.  Yields (column slice, [msy][block] byte index, in-payload
    mask)."""
    wh = width * height
    for x0 in range(0, msx, width):
        xs = np.arange(x0, min(x0 + width, msx), dtype=np.int64)
        idx = width * np.arange(msy, dtype=np.int64)[:, None] + xs[None, :]
        yield slice(x0, x0 + len(xs)), idx, idx < wh


def gmapping_publish(cells, width, height, last_writer=True):
    """PublishMap's loops (gmapping.cc:141-159) over storage classes [msy][msx]: x outer, y inner, into MAP_IDX =
    width * y + x of a width x height payload, a later write winning and bytes at or past width * height not written
    (unwritten bytes stay 0).  last_writer=False keeps the first write instead: the wrong rule, for premise tests."""
    msy, msx = cells.shape
    out = np.zeros(width * height, np.int8)
    blocks = list(_column_blocks(msx, msy, width, height))
    for xs, idx, keep in (blocks if last_writer else blocks[::-1]):
        out[idx[keep]] = cells[:, xs][keep]
    return out.reshape(height, width)


def gmapping_writers(msx, msy, width, height):
    """For every payload byte, the flat storage index (x + y * msx) of the cell PublishMap writes there last, and of
    the one it writes there first ([height][width], -1 for none)."""
    cell = np.arange(msx * msy, dtype=np.int64).reshape(msy, msx)
    out = []
    for order in (1, -1):
        w = np.full(width * height, -1, np.int64)
        for xs, idx, keep in list(_column_blocks(msx, msy, width, height))[::order]:
            w[idx[keep]] = cell[:, xs][keep]
        out.append(w.reshape(height, width))
    return tuple(out)


def gmapping_node(fields, params, ranges):
    """GMapping::ScanCallback on every scan of ranges [S][n] float32, fields = (angle_min, angle_increment, range_min,
    range_max).  -> (maps [k][height][width] int8, k = the first refused scan or S, the GMappingScan of every mapped
    scan)."""
    ranges = np.asarray(ranges, np.float32)
    width, height = gmapping_dims(params)
    angles = gmapping_angles(fields, ranges.shape[1])
    maps, scans = [], []
    for r in ranges:
        g = GMappingScan(params, angles, r)
        if g.refused:
            break
        maps.append(gmapping_publish(g.classes(params.occ_thresh), width, height))
        scans.append(g)
    out = np.stack(maps) if maps else np.zeros((0, height, width), np.int8)
    return out, len(maps), scans


# --------------------------------------------------------------------------------------------------------- Hector

BEGIN = (int(np.float32(800.0) + np.float32(0.5)), int(np.float32(800.0) + np.float32(0.5)))  # OccGridMapBase.h:182-192


def _log_odds(prob):
    """probToLogOdds (GridMapLogOdds.h:153-157)"""
    p = np.float32(prob)
    return np.float32(math.log(float(np.float32(p / (np.float32(1.0) - p)))))


LOG_ODDS_FREE, LOG_ODDS_OCC = _log_odds(0.4), _log_odds(0.6)  # GridMapLogOddsFunctions() (:98-102)


def hector_dims(params):
    """InitParams (hector_mapping.cc:57-58): map_size_ = (max - min) / resolution_, a float, truncated into ints."""
    res = float(np.float32(params.delta))
    return node_dim((params.xmax - params.xmin) / res), node_dim((params.ymax - params.ymin) / res)


def hector_points(fields, ranges):
    """ROSLaserScanToDataContainer (hector_mapping.cc:138-165): the float angle accumulated beam by beam, kept iff
    range_min < dist < range_max - 0.1f, the point Vector2f(cos(angle) * dist, sin(angle) * dist) of double products.
    -> float32 [k][2]."""
    angle, inc = np.float32(fields[0]), np.float32(fields[1])
    rmin, lim = np.float32(fields[2]), np.float32(fields[3]) - np.float32(0.1)
    pts = []
    for d in np.asarray(ranges, np.float32):
        if d > rmin and d < lim:
            pts.append((np.float32(math.cos(float(angle)) * float(d)), np.float32(math.sin(float(angle)) * float(d))))
        angle = np.float32(angle + inc)
    return np.array(pts, np.float32).reshape(-1, 2)


def hector_end_cell(p):
    """updateByScanJustOnce's end cell (OccGridMapBase.h:201-203): begin + (int)round(p / 0.05) on the float point."""
    return BEGIN[0] + int(c_round(float(p[0]) / 0.05)), BEGIN[1] + int(c_round(float(p[1]) / 0.05))


class HectorScan:
    """updateByScanJustOnce (OccGridMapBase.h:175-300) of one scan into a fresh GridMap of width x height, beam by
    beam: log-odds (float32) and update index per flat cell offset, kept sparsely (absent: 0.0f and -1).
    `beams` lists, per point, (end cell, drawn?, the flat offsets bresenham2D frees)."""

    def __init__(self, width, height, points):
        self.width, self.height = width, height
        self.lo, self.ui = {}, {}
        self.beams = []
        self.mark_free, self.mark_occ = 0 + 1, 0 + 2  # currUpdateIndex 0 (:177-178)
        for p in points:
            end = hector_end_cell(p)
            freed = []
            drawn = BEGIN != end and self._line(BEGIN, end, freed)
            self.beams.append((end, drawn, freed))

    def _inside(self, x, y):
        return 0 <= x < self.width and 0 <= y < self.height

    def _line(self, begin, end, freed):
        """updateLineBresenhami (:220-267); False where it returns without drawing."""
        (x0, y0), (x1, y1) = begin, end
        if not self._inside(x0, y0) or not self._inside(x1, y1):
            return False
        dx, dy = x1 - x0, y1 - y0
        sign = lambda v: 1 if v > 0 else -1  # util::sign
        off_dx, off_dy = sign(dx), sign(dy) * self.width
        start = y0 * self.width + x0
        if abs(dx) >= abs(dy):
            self._bresenham(abs(dx), abs(dy), abs(dx) // 2, off_dx, off_dy, start, freed)
        else:
            self._bresenham(abs(dy), abs(dx), abs(dy) // 2, off_dy, off_dx, start, freed)
        self._cell_occ(y1 * self.width + x1)
        return True

    def _bresenham(self, da, db, err, off_a, off_b, offset, freed):
        """bresenham2D (:270-299): the error walk, da cells from the begin cell."""
        self._cell_free(offset)
        freed.append(offset)
        for _ in range(da - 1):
            offset += off_a
            err += db
            if err >= da:
                offset += off_b
                err -= da
            self._cell_free(offset)
            freed.append(offset)

    def _cell_free(self, o):  # bresenhamCellFree (:302-312)
        if self.ui.get(o, -1) < self.mark_free:
            self.lo[o] = np.float32(self.lo.get(o, np.float32(0.0)) + LOG_ODDS_FREE)  # updateSetFree
            self.ui[o] = self.mark_free

    def _cell_occ(self, o):  # bresenhamCellOcc (:315-330)
        u = self.ui.get(o, -1)
        if u < self.mark_occ:
            v = self.lo.get(o, np.float32(0.0))
            if u == self.mark_free:
                v = np.float32(v - LOG_ODDS_FREE)  # updateUnsetFree
            if v < np.float32(50.0):  # updateSetOccupied
                v = np.float32(v + LOG_ODDS_OCC)
            self.lo[o] = v
            self.ui[o] = self.mark_occ

    def publish(self):
        """PublishMap (hector_mapping.cc:177-211): -1, then 0 where the log-odds are < 0, 100 where > 0."""
        out = np.full(self.width * self.height, -1, np.int8)
        for o, v in self.lo.items():
            if v < 0:
                out[o] = 0
            elif v > 0:
                out[o] = 100
        return out.reshape(self.height, self.width)


def hector_node(fields, params, ranges):
    """HectorMapping::ScanCallback on every scan -> (maps [S][height][width] int8, the HectorScan of every scan)."""
    width, height = hector_dims(params)
    maps, scans = [], []
    for r in np.asarray(ranges, np.float32):
        h = HectorScan(width, height, hector_points(fields, r))
        maps.append(h.publish())
        scans.append(h)
    out = np.stack(maps) if maps else np.zeros((0, height, width), np.int8)
    return out, scans
