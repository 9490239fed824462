"""Brute-force ray tracing for the Karto occupancy grid (K2c) and the GMapping hit/visit map (K2b).

Plain Python integer loops, one cell per iteration, written from the behaviour of the original project; the line numbers
cite lesson6/lib/open_karto/include/open_karto/Karto.h (and Math.h), lesson6/src/karto_slam.cc,
lesson4/src/gmapping/gmapping.cc and lesson4/include/lesson4/gmapping/grid/{map.h,harray2d.h,gridlinetraversal.h}.
It uses neither the closed-form line of the kernels, nor the C restatement under oracle/, nor numpy for the line walks,
so it checks all of them independently.  Floating-point steps keep the reference's operation order on Python floats
(IEEE doubles, no fused multiply-add) with the C library's math.cos / math.sin."""
from __future__ import annotations

import math

import numpy as np

# ---------------------------------------------------------------------------------------------------------- Karto

KT_TOLERANCE = 1e-06                 # Math.h:41
KT_PI = 3.14159265358979323846       # Math.h:32
KT_2PI = 6.28318530717958647692      # Math.h:33
BIG = 999999999999999999.99999       # BoundingBox2's empty box, Karto.h:2765
MIN_PASS_THROUGH = 2                 # OccupancyGrid's defaults, Karto.h:5632-5633
OCCUPANCY_THRESHOLD = 0.1
UNKNOWN, OCCUPIED, FREE = 0, 100, 255  # GridStates, Karto.h:4195-4197


def karto_round(v: float) -> int:
    """math::Round (Math.h:87-90): halves away from zero, as floor(v + 0.5) / ceil(v - 0.5) on doubles."""
    return math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5)


def normalize_angle(a: float) -> float:
    """math::NormalizeAngle (Math.h:182-211)"""
    while a < -KT_PI:
        a = a + int(a / -KT_2PI) * KT_2PI if a < -KT_2PI else a + KT_2PI
    while a > KT_PI:
        a = a - int(a / KT_2PI) * KT_2PI if a > KT_2PI else a - KT_2PI
    return a


def sensor_pose(robot, offset):
    """LocalizedRangeScan::GetSensorAt = Transform(robot).TransformPose(offset) (Karto.h:5310-5313).

    Transform(Pose2(), robot): identity when robot == Pose2() (:2911-2917), else the rotation
    Matrix3::FromAxisAngle(0, 0, 1, heading) (:2392-2421) and the translation robot - Pose2() (:2920-2934).
    TransformPose (:2881-2887) adds the rotated offset, Matrix3 * Pose2 summing left to right (:2574-2583)."""
    rx, ry, rh = (float(v) for v in robot)
    ox, oy, oh = (float(v) for v in offset)
    if rx == 0.0 and ry == 0.0 and rh == 0.0:
        m00, m01, m02, m10, m11, m12 = 1.0, 0.0, 0.0, 0.0, 1.0, 0.0
        tx, ty, th = 0.0, 0.0, 0.0
    else:
        radians = rh - 0.0
        c, s = math.cos(radians), math.sin(radians)
        omc = 1.0 - c
        ax, ay, az = 0.0, 0.0, 1.0
        m00 = ax * ax * omc + c
        m01 = ax * ay * omc - az * s
        m02 = ax * az * omc + ay * s
        m10 = ax * ay * omc + az * s
        m11 = ay * ay * omc + c
        m12 = ay * az * omc - ax * s
        tx, ty, th = rx, ry, rh - 0.0
    x = tx + (m00 * ox + m01 * oy + m02 * oh)
    y = ty + (m10 * ox + m11 * oy + m12 * oh)
    return x, y, normalize_angle(oh + th)


def point_readings(laser, ranges, robot):
    """LocalizedRangeScan::Update, the unfiltered list (Karto.h:5379-5401): one point per reading."""
    sx, sy, sh = sensor_pose(robot, laser.offset_pose)
    pts = []
    for i in range(laser.n_readings):
        r = float(ranges[i])
        angle = sh + laser.min_angle + float(i) * laser.angular_resolution
        pts.append((sx + (r * math.cos(angle)), sy + (r * math.sin(angle))))
    return (sx, sy), pts


def in_range(v, a, b):
    """math::InRange (Math.h:172-175)"""
    return v >= a and v <= b


def scan_bbox(laser, ranges, robot):
    """The scan's BoundingBox2 (Karto.h:5418-5424): sensor position plus the points whose reading is
    InRange(minimum range, range threshold) (:5382); Add keeps the running minimum and maximum (:2815-2819, 987-1005)."""
    (sx, sy), pts = point_readings(laser, ranges, robot)
    mn, mx = [BIG, BIG], [-BIG, -BIG]

    def add(x, y):
        if x < mn[0]:
            mn[0] = x
        if y < mn[1]:
            mn[1] = y
        if x > mx[0]:
            mx[0] = x
        if y > mx[1]:
            mx[1] = y

    add(sx, sy)
    for i, (x, y) in enumerate(pts):
        if in_range(float(ranges[i]), laser.min_range, laser.range_threshold):
            add(x, y)
    return [mn[0], mn[1], mx[0], mx[1]]


def union_bbox(laser, ranges, poses):
    """OccupancyGrid::ComputeDimensions' box (Karto.h:5810-5814): BoundingBox2::Add(box) = Add(min); Add(max)
    (:2824-2828)."""
    mn, mx = [BIG, BIG], [-BIG, -BIG]
    for s in range(len(poses)):
        b = scan_bbox(laser, ranges[s], poses[s])
        for x, y in ((b[0], b[1]), (b[2], b[3])):
            if x < mn[0]:
                mn[0] = x
            if y < mn[1]:
                mn[1] = y
            if x > mx[0]:
                mx[0] = x
            if y > mx[1]:
                mx[1] = y
    return [mn[0], mn[1], mx[0], mx[1]]


def trace_line(x0, y0, x1, y1):
    """Grid::TraceLine (Karto.h:4680-4745): every cell of the line in visiting order, in the grid or not, walked with
    the error accumulator."""
    steep = abs(y1 - y0) > abs(x1 - x0)
    if steep:
        x0, y0, x1, y1 = y0, x0, y1, x1
    if x0 > x1:
        x0, x1, y0, y1 = x1, x0, y1, y0
    delta_x, delta_y = x1 - x0, abs(y1 - y0)
    error, y = 0, y0
    ystep = 1 if y0 < y1 else -1
    cells = []
    for x in range(x0, x1 + 1):
        cells.append((y, x) if steep else (x, y))
        error += delta_y
        if 2 * error >= delta_x:
            y += ystep
            error -= delta_x
    return cells


def update_cell(passes: int, hits: int) -> int:
    """OccupancyGrid::UpdateCell (Karto.h:5953-5968) on an unknown (cleared) cell."""
    if passes > MIN_PASS_THROUGH:
        return OCCUPIED if float(hits) / float(passes) > OCCUPANCY_THRESHOLD else FREE
    return UNKNOWN


def update(passes, hits):
    """OccupancyGrid::Update (Karto.h:5973-5990) over every counter, padding columns included: update_cell on whole
    arrays (the same double division and comparisons)."""
    p, h = passes.astype(np.float64), hits.astype(np.float64)
    ratio = h / np.where(passes > 0, p, 1.0)
    return np.where(passes > MIN_PASS_THROUGH, np.where(ratio > OCCUPANCY_THRESHOLD, OCCUPIED, FREE),
                    UNKNOWN).astype(np.uint8)


def occupancy_grid(laser, ranges, poses, resolution, bbox=None):
    """OccupancyGrid::CreateFromScans (Karto.h:5828-5843), or with an explicit `bbox` {min x, min y, max x, max y} a
    grid of that box fed with these scans (a grid can then be smaller than its rays).  Returns the same dict as
    oracle.port.occupancy_grid, with cell_visits = in-grid counter increments (pass per line cell, pass + hit at a
    valid end point)."""
    ranges = np.asarray(ranges, np.float64).reshape(-1, laser.n_readings)
    poses = np.asarray(poses, np.float64).reshape(-1, 3)
    if bbox is None:
        bbox = union_bbox(laser, ranges, poses)
    scale = 1.0 / resolution
    width = int(karto_round((bbox[2] - bbox[0]) * scale))  # ComputeDimensions (:5816-5821)
    height = int(karto_round((bbox[3] - bbox[1]) * scale))
    step = (width + 7) & ~7  # math::AlignValue(width, 8) (:4442)
    off_x, off_y = float(bbox[0]), float(bbox[1])
    passes, hits = [0] * (step * height), [0] * (step * height)
    visits = 0

    def to_grid(x, y):  # CoordinateConverter::WorldToGrid (:4237-4252), flipY false
        return int(karto_round((x - off_x) * scale)), int(karto_round((y - off_y) * scale))

    threshold, max_range, min_range = laser.range_threshold, laser.max_range, laser.min_range
    for s in range(len(poses)):
        (sx, sy), pts = point_readings(laser, ranges[s], poses[s])
        for i in range(laser.n_readings):  # AddScan (:5852-5899)
            px, py = pts[i]
            rr = float(ranges[s, i])
            end_valid = rr < (threshold - KT_TOLERANCE)
            if rr <= min_range or rr >= max_range or math.isnan(rr):
                continue
            elif rr >= threshold:
                ratio = threshold / rr
                dx, dy = px - sx, py - sy
                px, py = sx + ratio * dx, sy + ratio * dy
            # RayTrace (:5910-5945)
            fx, fy = to_grid(sx, sy)
            tx, ty = to_grid(px, py)
            for cx, cy in trace_line(fx, fy, tx, ty):
                if 0 <= cx < width and 0 <= cy < height:  # IsValidGridIndex
                    passes[cx + cy * step] += 1
                    visits += 1
            if end_valid and 0 <= tx < width and 0 <= ty < height:
                passes[tx + ty * step] += 1
                hits[tx + ty * step] += 1
                visits += 2
    pa = np.array(passes, np.int64).astype(np.uint32).reshape(height, step)
    hi = np.array(hits, np.int64).astype(np.uint32).reshape(height, step)
    return dict(width=width, height=height, width_step=step, offset=np.array([off_x, off_y]), cell_visits=visits,
                passes=pa, hits=hi, cells=update(pa, hi))


def karto_ros_map(cells, width, height):
    """SlamKarto::updateMap's payload (karto_slam.cc:546-569): row-major width x height, unknown -1, occupied 100,
    free 0."""
    value = np.zeros(256, np.int8)
    value[UNKNOWN], value[OCCUPIED], value[FREE] = -1, 100, 0
    assert np.isin(cells, (UNKNOWN, OCCUPIED, FREE)).all()
    return value[np.asarray(cells)[:height, :width]]


# ------------------------------------------------------------------------------------------------------- GMapping

PATCH_MAGNITUDE = 5  # HierarchicalArray2D's default (harray2d.h:36)


def c_round(v: float) -> int:
    """C round(): halves away from zero, exactly (the integer part of a double is exact)."""
    t = math.trunc(v)
    if abs(v - t) >= 0.5:
        t += 1 if v > 0 else -1
    return t


def gmap_layout(xmin, ymin, xmax, ymax, delta):
    """Map ctor (map.h:133-140): 32-cell patch storage over ceil(size / delta) cells, and the half sizes.
    Returns (centre x, centre y, mapSizeX, mapSizeY, sizeX2, sizeY2); the centre is gmapping.cc:130-132's."""
    cx, cy = (xmin + xmax) / 2.0, (ymin + ymax) / 2.0
    xs, ys = int(math.ceil((xmax - xmin) / delta)), int(math.ceil((ymax - ymin) / delta))
    msx = (xs >> PATCH_MAGNITUDE) << PATCH_MAGNITUDE  # harray2d.h:75-76, map.h:136-137
    msy = (ys >> PATCH_MAGNITUDE) << PATCH_MAGNITUDE
    return cx, cy, msx, msy, int(c_round((cx - xmin) / delta)), int(c_round((cy - ymin) / delta))


def grid_line(start, end):
    """GridLineTraversal::gridLine (gridlinetraversal.h:27-207): gridLineCore's midpoint walk from the end with the
    smaller dominant coordinate, reversed when it did not begin at `start`."""
    (sx, sy), (ex, ey) = start, end
    dx, dy = abs(ex - sx), abs(ey - sy)
    pts = []
    if dy <= dx:
        d, incr1, incr2 = 2 * dy - dx, 2 * dy, 2 * (dy - dx)
        if sx > ex:
            x, y, ydirflag, xend = ex, ey, -1, sx
        else:
            x, y, ydirflag, xend = sx, sy, 1, ex
        pts.append((x, y))
        ystep = 1 if (ey - sy) * ydirflag > 0 else -1
        while x < xend:
            x += 1
            if d < 0:
                d += incr1
            else:
                y += ystep
                d += incr2
            pts.append((x, y))
    else:
        d, incr1, incr2 = 2 * dx - dy, 2 * dx, 2 * (dx - dy)
        if sy > ey:
            y, x, yend, xdirflag = ey, ex, sy, -1
        else:
            y, x, yend, xdirflag = sy, sx, ey, 1
        pts.append((x, y))
        xstep = 1 if (ex - sx) * xdirflag > 0 else -1
        while y < yend:
            y += 1
            if d < 0:
                d += incr1
            else:
                x += xstep
                d += incr2
            pts.append((x, y))
    if pts[0] != (sx, sy):
        pts.reverse()
    return pts


class GMapReference:
    """ScanMatcherMap as GMapping::ComputeMap / PublishMap use it (gmapping.cc:127-242), with the laser at
    `laser_xy` (heading 0; beam angles absolute).  A call in which a kept beam's end cell lies outside the storage —
    where the original asserts (map.h:186-191) — returns -1 and changes nothing, as the library defines it."""

    def __init__(self, xmin, ymin, xmax, ymax, delta):
        self.bounds = (xmin, ymin, xmax, ymax, delta)
        self.cx, self.cy, self.size_x, self.size_y, self.sx2, self.sy2 = gmap_layout(xmin, ymin, xmax, ymax, delta)
        c = self.size_x * self.size_y
        self.n, self.visits = [0] * c, [0] * c
        self.acc_x, self.acc_y = [np.float32(0)] * c, [np.float32(0)] * c
        self.acc64_x, self.acc64_y = [0.0] * c, [0.0] * c  # float64 sums of the float32 hit coordinates
        self.abs64 = [0.0] * c  # float64 sums of |hit coordinate| (bounds the float32 summation error)

    def world2map(self, x, y):  # map.h:171-174
        d = self.bounds[4]
        return int(c_round((x - self.cx) / d)) + self.sx2, int(c_round((y - self.cy) / d)) + self.sy2

    def inside(self, p):
        return 0 <= p[0] < self.size_x and 0 <= p[1] < self.size_y

    def compute_map(self, ranges, angles, laser_xy=(0.0, 0.0), max_range=30 - 0.01, max_urange=25.0):
        lx, ly = float(laser_xy[0]), float(laser_xy[1])
        p0 = self.world2map(lx, ly)
        if not self.inside(p0):
            return -1
        lines, hit_list = [], []
        for i in range(len(ranges)):
            d = float(ranges[i])
            if d > max_range or d == 0.0 or not math.isfinite(d):  # gmapping.cc:193-195
                continue
            if d > max_urange:
                d = max_urange
            hx, hy = lx, ly
            hx += d * math.cos(float(angles[i]))
            hy += d * math.sin(float(angles[i]))
            p1 = self.world2map(hx, hy)
            if not self.inside(p1):
                return -1
            lines.append(grid_line(p0, p1))
            if d < max_urange:  # gmapping.cc:218-223
                hit_list.append((hx, hy))
        sx = self.size_x
        for line in lines:  # all points but the last are free (gmapping.cc:229-235)
            for k in range(len(line) - 1):
                x, y = line[k]
                self.visits[x + y * sx] += 1
        for hx, hy in hit_list:  # PointAccumulator::update(true, hit) (gmapping.cc:237-241, map.h:37-48)
            x, y = self.world2map(hx, hy)
            c = x + y * sx
            fx, fy = np.float32(hx), np.float32(hy)
            self.acc_x[c] = np.float32(self.acc_x[c] + fx)
            self.acc_y[c] = np.float32(self.acc_y[c] + fy)
            self.acc64_x[c] += float(fx)
            self.acc64_y[c] += float(fy)
            self.abs64[c] += max(abs(float(fx)), abs(float(fy)))
            self.n[c] += 1
            self.visits[c] += 1
        return 0

    def cells(self):
        sh = (self.size_y, self.size_x)
        return (np.array(self.n, np.int32).reshape(sh), np.array(self.visits, np.int32).reshape(sh),
                np.array(self.acc_x, np.float32).reshape(sh), np.array(self.acc_y, np.float32).reshape(sh))

    def ros_map(self, occ_thresh=0.25):
        """GMapping::PublishMap (gmapping.cc:141-159): x outer, y inner, into MAP_IDX = width * y + x of a
        width x height array (width = (uint32)((xmax - xmin) / resolution), gmapping.cc:72); a later write to the
        same byte wins and bytes past the end are not written."""
        xmin, ymin, xmax, ymax, delta = self.bounds
        width, height = int((xmax - xmin) / delta), int((ymax - ymin) / delta)
        out = [0] * (width * height)
        for x in range(self.size_x):
            for y in range(self.size_y):
                c = x + y * self.size_x
                v = self.visits[c]
                occ = float(self.n[c]) * 1 / float(v) if v else -1.0  # PointAccumulator::operator double (map.h:27)
                o = width * y + x
                if o >= width * height:
                    continue
                out[o] = -1 if occ < 0 else (100 if occ > occ_thresh else 0)
        return np.array(out, np.int8).reshape(height, width)
