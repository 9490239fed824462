"""A float64 restatement of the Hector Gauss-Newton scan match (CPU only, numpy), the yardstick of the fast device paths
(tests/test_gpu_hector_fast.py) and checked itself against the float32 restatement by tests/test_hector_gn_reference.py.
The file name keeps pytest from collecting it; tests import it.

It follows the same formulas as the float32 restatement (oracle/hector_oracle.c) and hector_grid.cuh, with every
operation after the map transform in float64:
- the map transform of a level: the float32 constants of MapRepMultiMap's pyramid (cell length res * 2^l, the level-0
  offset for every level, points scaled by 2^-l), applied in float64;
- getGridProbability: exp of the float32 log-odds in float64;
- interpMapValueWithDerivatives: the bounds rule x < 0 | x > sx - 2 | y < 0 | y > sy - 2 -> zeros, then the bilinear
  value and gradient of the four cells (a NaN coordinate reads cell 0 and carries its NaN through the fractions);
- getCompleteHessianDerivs: the nine sums H00 H11 H22 H01 H02 H12 and dTr, and for each the sum of the absolute values of
  its terms (the scale of the float32 rounding of that sum);
- estimateTransformationLogLh: the cofactor solve of H dir = dTr and the +-0.2 rad clamp of the heading step;
- ScanMatcher::matchData on one level and MapRepMultiMap::matchData over the pyramid (1 + 3 iterations per coarse level,
  1 + 5 on level 0).

Map poses are (x, y, heading) in level cells; world poses in metres."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

F = np.float32
COARSE_ITERATIONS, FINE_ITERATIONS = 3, 5


@dataclass
class Level:
    """One map level: probabilities in float64 and the float32 transform constants of GridMapBase."""
    prob: np.ndarray  # [sy, sx] float64
    tw_lin: float     # world -> map: map = tw_lin * world + (tw_tx, tw_ty)
    tw_tx: float
    tw_ty: float
    wt_lin: float     # map -> world, as GridMapBase's Affine inverse (float32)
    wt_tx: float
    wt_ty: float

    @property
    def sx(self):
        return self.prob.shape[1]

    @property
    def sy(self):
        return self.prob.shape[0]

    def map_coords32(self, world):
        """getMapCoordsPose in float32, operation for operation: the map pose a float32 implementation starts from."""
        wx, wy = F(world[0]), F(world[1])
        mx = (F(self.tw_lin) * wx + F(0) * wy) + F(self.tw_tx)
        my = (F(0) * wx + F(self.tw_lin) * wy) + F(self.tw_ty)
        return np.array([mx, my, F(world[2])], np.float32)

    def map_coords(self, world):
        return np.array([self.tw_lin * world[0] + self.tw_tx, self.tw_lin * world[1] + self.tw_ty, world[2]], np.float64)

    def world_coords(self, m):
        return np.array([(m[0] - self.tw_tx) / self.tw_lin, (m[1] - self.tw_ty) / self.tw_lin, m[2]], np.float64)


def grid_probability(log_odds):
    odds = np.exp(np.asarray(log_odds, np.float32).astype(np.float64))
    return odds / (odds + 1.0)


def make_level(log_odds, resolution, size_x, size_y, start, level):
    """Level `level` of a processor created with (resolution, size_x, size_y, start): its log-odds plane [sy >> l,
    sx >> l] (float32) and the transform of hector_grid.cuh's map_transform with MapRepMultiMap's offset."""
    lo = np.asarray(log_odds, np.float32)
    assert lo.shape == (size_y >> level, size_x >> level), (lo.shape, size_x, size_y, level)
    off_x = F(F(resolution) * F(size_x)) * F(start[0])
    off_y = F(F(resolution) * F(size_y)) * F(start[1])
    cell = F(resolution)
    for _ in range(level):
        cell = cell * F(2)
    tw_lin = F(1) / cell
    tw_tx, tw_ty = tw_lin * off_x, tw_lin * off_y
    invdet = F(1) / (tw_lin * tw_lin - F(0) * F(0))
    i01 = F(-0.0) * invdet
    wt_lin = tw_lin * invdet
    wt_tx = -(wt_lin * tw_tx + i01 * tw_ty)
    wt_ty = -(i01 * tw_tx + wt_lin * tw_ty)
    return Level(grid_probability(lo), float(tw_lin), float(tw_tx), float(tw_ty), float(wt_lin), float(wt_tx),
                 float(wt_ty))


def processor_levels(proc, resolution, size_x, size_y, start, levels, **_):
    """Every level of a PortHectorProcessor (or a device handle with .level(i)), coarsest last."""
    return [make_level(proc.level(l)[0], resolution, size_x, size_y, start, l) for l in range(levels)]


def interp(level, x, y, cells=False):
    """interpMapValueWithDerivatives at map coordinates x, y (arrays): value, d/dx, d/dy (float64), and with `cells`
    the flat index of each point's cell (-1 outside)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    outside = (x < 0) | (x > level.sx - 2) | (y < 0) | (y > level.sy - 2)
    with np.errstate(invalid="ignore"):
        ix = np.where(outside | np.isnan(x), 0, np.trunc(np.nan_to_num(x))).astype(np.int64)
        iy = np.where(outside | np.isnan(y), 0, np.trunc(np.nan_to_num(y))).astype(np.int64)
        fx, fy = x - ix, y - iy
        p = level.prob
        i0, i1, i2, i3 = p[iy, ix], p[iy, ix + 1], p[iy + 1, ix], p[iy + 1, ix + 1]
        xfi, yfi = 1.0 - fx, 1.0 - fy
        val = (i0 * xfi + i1 * fx) * yfi + (i2 * xfi + i3 * fx) * fy
        gx = -((i0 - i1) * yfi + (i2 - i3) * fy)
        gy = -((i0 - i2) * xfi + (i1 - i3) * fx)
    z = np.zeros_like(val)
    out = np.where(outside, z, val), np.where(outside, z, gx), np.where(outside, z, gy)
    return out + (np.where(outside, -1, iy * level.sx + ix),) if cells else out


@dataclass
class Sums:
    H: np.ndarray       # [3, 3]
    dTr: np.ndarray     # [3]
    H_abs: np.ndarray   # [3, 3]: the sum of |term| of each entry
    dTr_abs: np.ndarray
    H_floor: np.ndarray  # [3, 3]: the sum of the terms' absolute error floors (GRADIENT_ERROR)


UPPER = ((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2))
# The absolute error of a float32 gradient: a difference of float32 probabilities (each within an ulp of a value below
# 1, 2^-24, and the device's expf another ulp) times fractions below 1.  A gradient near zero has no relative accuracy
# at all, so the H terms it enters carry this floor (times the other factor) besides their relative rounding.
GRADIENT_ERROR = 2.0 ** -22


def point_terms(level, pose, pts, cells=False, floors=False):
    """The per-point terms of getCompleteHessianDerivs at map pose `pose` (x, y in level cells, heading) for points
    `pts` [n, 2] in level cells (already scaled to the level): dTr [3, n] and the six distinct H entries [6, n] in the
    order of UPPER (and with `cells` each point's cell, see interp; with `floors` each H term's absolute error floor,
    see GRADIENT_ERROR)."""
    p = np.asarray(pts, np.float64).reshape(-1, 2)
    px, py = p[:, 0], p[:, 1]
    th = float(pose[2])
    c, s = math.cos(th), math.sin(th)
    val, t1, t2, cell = interp(level, (c * px - s * py) + float(pose[0]), (s * px + c * py) + float(pose[1]), True)
    fun = 1.0 - val
    rot = (-s * px - c * py) * t1 + (c * px - s * py) * t2
    out = np.stack([t1 * fun, t2 * fun, rot * fun]), np.stack([t1 * t1, t2 * t2, rot * rot, t1 * t2, t1 * rot, t2 * rot])
    if cells:
        out = out + (cell,)
    if floors:
        e = GRADIENT_ERROR * (cell >= 0)
        er = e * (np.abs(-s * px - c * py) + np.abs(c * px - s * py))
        a1, a2, ar = np.abs(t1), np.abs(t2), np.abs(rot)
        out = out + (np.stack([2 * a1 * e, 2 * a2 * e, 2 * ar * er, a1 * e + a2 * e, a1 * er + ar * e, a2 * er + ar * e]),)
    return out


def _sym(six):
    H = np.zeros((3, 3))
    for q, (i, j) in enumerate(UPPER):
        H[i, j] = H[j, i] = six[q]
    return H


def hessian_sums(level, pose, pts):
    """getCompleteHessianDerivs at map pose `pose` for level-scaled points `pts` [n, 2]."""
    d, h, fl = point_terms(level, pose, pts, floors=True)
    with np.errstate(invalid="ignore"):
        return Sums(_sym(h.sum(1)), d.sum(1), _sym(np.abs(h).sum(1)), np.abs(d).sum(1), _sym(fl.sum(1)))


def gn_step(H, dTr):
    """estimateTransformationLogLh's update: H^-1 dTr by cofactors (a singular H gives inf / NaN, as in float32), the
    heading step clamped to +-0.2 rad.  None where H00 or H11 is zero (no step)."""
    m = np.asarray(H, np.float64).reshape(9)
    if m[0] == 0.0 or m[4] == 0.0:
        return None
    with np.errstate(divide="ignore", invalid="ignore"):
        c00, c10, c20 = m[4] * m[8] - m[5] * m[7], m[5] * m[6] - m[3] * m[8], m[3] * m[7] - m[4] * m[6]
        det = c00 * m[0] + c10 * m[1] + c20 * m[2]
        inv = np.array([[c00, m[2] * m[7] - m[1] * m[8], m[1] * m[5] - m[2] * m[4]],
                        [c10, m[0] * m[8] - m[2] * m[6], m[2] * m[3] - m[0] * m[5]],
                        [c20, m[1] * m[6] - m[0] * m[7], m[0] * m[4] - m[1] * m[3]]]) / det
        d = inv @ np.asarray(dTr, np.float64)
    if d[2] > 0.2:
        d[2] = 0.2
    elif d[2] < -0.2:
        d[2] = -0.2
    return d


def normalize_angle(a):
    a = math.fmod(math.fmod(a, 2 * math.pi) + 2 * math.pi, 2 * math.pi)
    return a - 2 * math.pi if a > math.pi else a


@dataclass
class Match:
    pose: np.ndarray       # world pose after the match (float64)
    sums: Sums | None      # the last evaluation (None when no point was given)
    sums_pose: np.ndarray  # the map pose of that evaluation (level 0 for the pyramid)
    last_step: float       # largest |component| of the last Gauss-Newton step (cells, rad); 0 when none was taken
    singular: bool = False  # a step was taken through a (numerically) singular H: its result is rounding noise


def _singular(H):
    """H has H00, H11 != 0 (a step is taken) but a determinant below 1e-12 of the product of its diagonal."""
    d = abs(np.linalg.det(H)) if np.isfinite(H).all() else math.nan
    return not d >= 1e-12 * abs(H[0, 0] * H[1, 1] * H[2, 2])


def match_level(level, pts, begin_world, iterations):
    """ScanMatcher::matchData on one level: 1 + `iterations` evaluations from `begin_world`."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    if len(pts) == 0:
        return Match(np.asarray(begin_world, np.float64), None, None, 0.0)
    est = level.map_coords(np.asarray(begin_world, np.float64))
    sums, at, last, singular = None, est, 0.0, False
    for _ in range(1 + iterations):
        at = est.copy()
        sums = hessian_sums(level, at, pts)
        d = gn_step(sums.H, sums.dTr)
        last = 0.0 if d is None else float(np.max(np.abs(d))) if np.isfinite(d).all() else math.inf
        if d is not None:
            singular = singular or _singular(sums.H)
            est = est + d
    est[2] = normalize_angle(est[2]) if np.isfinite(est[2]) else est[2]
    return Match(level.world_coords(est), sums, at, last, singular)


def match_pyramid(levels, pts, hint_world):
    """MapRepMultiMap::matchData: levels coarsest first, each from the previous level's world pose; the points of level
    l are the level-0 points times 2^-l (exact in float32).  `singular` covers every level."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    pose = np.asarray(hint_world, np.float32).astype(np.float64)
    m, singular = None, False
    for l in range(len(levels) - 1, -1, -1):
        m = match_level(levels[l], pts * F(2.0 ** -l), pose, FINE_ITERATIONS if l == 0 else COARSE_ITERATIONS)
        singular = singular or m.singular
        pose = m.pose
    m.singular = singular
    return m


def converged(m, tol=1e-6):
    """The float64 match's last level-0 step is below `tol` (cells / rad) and no step went through a singular H."""
    return m.sums is not None and not m.singular and m.last_step < tol


def hessian_at(level, pts, map_pose):
    return hessian_sums(level, map_pose, np.asarray(pts, np.float32).reshape(-1, 2))


def pose_slack(level, pts, world):
    """How far the six H sums can move over the rounding of a pose recovered from a float32 world pose.

    The last H of a match is evaluated at the map pose before the final step, and the caller only has the world pose
    after it: even where that step is below the float32 grid, get_world_coords / get_map_coords round by about one ulp
    of each coordinate, and normalize_angle moves a negative heading by up to half an ulp of heading + 2pi.  Inside a
    cell the sums move smoothly, by about that relative amount; but a point that lies within that distance of a cell
    edge may be evaluated in the neighbouring cell, where its gradient jumps.  Over the 8 corners of the box
    (x, y +- dxy, heading +- dth) around the recovered pose: the largest signed change of each sum over the points that
    stay in their cells, plus, for each point that changes cells at some corner, its largest change.
    Returns (recovered map pose, slack [3, 3])."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    m = level.map_coords32(world)
    w = np.asarray(world, np.float32)
    dxy = 0.5 * (np.spacing(np.abs(m[:2])).max() + float(level.tw_lin) * np.spacing(np.abs(w[:2])).max())
    dth = 0.5 * float(np.spacing(F(2 * np.pi)))
    _, h0, c0 = point_terms(level, m, pts, cells=True)
    corners = []
    for sx in (-1, 1):
        for sy in (-1, 1):
            for st in (-1, 1):
                _, h, c = point_terms(level, (m[0] + sx * dxy, m[1] + sy * dxy, float(m[2]) + st * dth), pts, cells=True)
                corners.append((h - h0, c != c0))
    moved = np.any([f for _, f in corners], axis=0)
    smooth = np.max([np.abs(d[:, ~moved].sum(1)) for d, _ in corners], axis=0)
    jumps = np.max([np.abs(d[:, moved]) for d, _ in corners], axis=0).sum(1) if moved.any() else 0.0
    return m, _sym(smooth + jumps)


def hessian_excess(H32, sums, slack=None):
    """max over the six distinct entries of |H32 - H64| - floor - slack, in units of sum|term| (the float32 rounding
    scale; floor = Sums.H_floor):
    an entry meets the bound k * sum|term| + floor + slack where this is <= k.  0 where an entry's terms are all zero and the
    float32 entry is zero too; inf where they are zero and it is not, or where H32 is not finite."""
    H32 = np.asarray(H32, np.float64).reshape(3, 3)
    slack = np.zeros((3, 3)) if slack is None else slack
    r = 0.0
    for i, j in UPPER:
        d, a = abs(H32[i, j] - sums.H[i, j]), sums.H_abs[i, j]
        if not np.isfinite(d):
            return math.inf
        d = max(d - slack[i, j] - sums.H_floor[i, j], 0.0)
        r = max(r, d / a if a > 0 else (0.0 if d == 0 else math.inf))
    return r


def angle_diff(a, b):
    return (np.asarray(a, np.float64) - np.asarray(b, np.float64) + np.pi) % (2 * np.pi) - np.pi


# ---- the matched cases: fixed maps, scans matched from their hints ----

GATE_SHUT = dict(min_dist=1e9, min_angle=1e9)


def warm_scans(stream, family):
    """The four scans that build the maps: the longest of the `long` family (its last), else the first four."""
    idx = range(len(stream) - 4, len(stream)) if family == "long" else range(4)
    return [stream.scans[i] for i in idx], stream.hints[list(idx)]


def warm_up(proc, stream, family):
    """Maps for a processor whose gate stays shut, the same in exact and fast mode: each warm scan is matched once (which
    fills the coarse levels' point containers, MapRepMultiMap::updateByScan draws the coarse levels from them) and
    then drawn at its hint with map_without_matching.  Only the first match moves a map: the gate opens on the first
    scan, where every map is empty, so no step is taken.  Works on the restatement and on a single device handle."""
    scans, hints = warm_scans(stream, family)
    for i in range(len(scans)):
        proc.update(scans[i], (0, 0), hints[i])
        proc.update(scans[i], (0, 0), hints[i], True)


# the bound of a float32 H sum: K * sum|term| (+ pose_slack where the evaluation pose is recovered from a world pose);
# chosen and justified in tests/test_hector_gn_reference.py
K = 1e-5
MIN_POSE_POINTS = 575  # below this a near-singular Hessian may send the float32 sums down another path (1e-4 poses)


@dataclass
class Case:
    stream: object
    kw: dict
    levels: list        # the float64 levels of the warmed-up maps
    poses: np.ndarray   # the restatement's poses [n, 3]
    covs: np.ndarray    # and Hessians [n, 3, 3]
    flags: np.ndarray   # and gate decisions [n]
    matches: list       # the float64 matches (match_pyramid) from the same hints


def cpu_case(geometry, family):
    """One geometry and family of tests/hector_cases.py on the restatement (gate shut, warmed up, matched from the
    hints) and on the float64 reference."""
    import hector_cases as hc
    from oracle import port
    kw = dict(hc.processor_kw(geometry), **GATE_SHUT)
    s = hc.make_stream(geometry, family)
    c = port.PortHectorProcessor(**kw)
    warm_up(c, s, family)
    levels = processor_levels(c, **kw)
    p, cv, f = hc.run_stream(c, s, "hints")
    c.close()
    return Case(s, kw, levels, p, cv, f, [match_pyramid(levels, pts, s.hints[i]) for i, pts in enumerate(s.scans)])


def check_hessian(case, i, H32, world32):
    """H32, the last Hessian of a float32 match of scan i that ended at world32, against the float64 sums at the
    recovered pose.  Returns the excess over K * sum|term| + pose_slack in units of sum|term| (<= K passes), or None
    where the float64 match did not converge (the last H was evaluated a visible step away from the result)."""
    if not converged(case.matches[i]):
        return None
    pts = case.stream.scans[i]
    mp, slack = pose_slack(case.levels[0], pts, world32)
    return hessian_excess(H32, hessian_at(case.levels[0], pts, mp), slack)


def pose_error(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(max(np.abs(a[:2] - b[:2]).max(), abs(angle_diff(a[2], b[2]))))
