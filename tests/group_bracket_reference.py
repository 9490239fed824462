"""The group pass of the correlative sweep's angle bound (k_sweep_bound<., BOUND_GROUPS> in csrc/karto_matcher.cu)
restated in numpy float32, and the group bound gub it yields.

For each beam and each group of BOUND_GROUP consecutive angles the kernel brackets the beam's lookup values per axis
in fp32: cf, sf = (float)cos, (float)sin of the member angles, x = cf px - sf py and y = sf px + cf py of the fp32
scan-local point, the smallest and largest over the members scaled and widened by the margin
mg_match + 1e-5 (|px| + |py|) scale, mg_match = 4e-3 + 1e-15 (|gox| + |goy|) scale, and rounded outwards to
[ceil(lo - 0.5), floor(hi + 0.5)].  A bracket end at 8192 cells or more, a non-finite point, or a spread of more than
BOUND_SPREAD cells on an axis sends the beam to the per-member fallback (the largest P7 over the members' exact
origins, members whose window lies wholly outside the grid adding 0); otherwise the beam adds P7 at the bracket's low
corner, whose class is 0 (in the pooled planes), 4 (read with the range test) or 255 (every corner outside: 0).

The library is built with -fmad=false, so numpy's IEEE float32 operations are the kernel's.  The device's cos and sin
may differ from the C library's in the last place: `Brackets.borderline` marks the (group, beam) pairs whose result
could depend on that, a bracket end within BORDER cells of a rounding boundary or of 8192, or a member angle whose
(float)cos / (float)sin changes when the double moves by one unit in the last place."""
import math

import numpy as np

from test_prune_bound import INVALID, penalties
from test_prune_group_bound import GROUP, SPREAD, pooled7

LIMIT = 8192.0   # bracket ends at or past this many cells take the fallback
BORDER = 1e-6    # cells: a bracket end this close to a rounding boundary is borderline
SPAN = 31        # window rows - 1 of a pruned sweep (one 32 x 32 tile)
f32 = np.float32


def kround(v):
    """math::Round: half away from zero"""
    return np.where(v >= 0.0, np.floor(v + 0.5), np.ceil(v - 0.5))


def local_points(pts, sensor_pose):
    """the scan-local points GridIndexLookup::ComputeOffsets rotates (Transform(sensorPose).InverseTransformPose)"""
    pts = np.asarray(pts, dtype=np.float64)
    if sensor_pose[0] == 0.0 and sensor_pose[1] == 0.0 and sensor_pose[2] == 0.0:
        return pts[:, 0].copy(), pts[:, 1].copy()
    r = 0.0 - sensor_pose[2]
    c, s = math.cos(r), math.sin(r)
    dx, dy = pts[:, 0] - sensor_pose[0], pts[:, 1] - sensor_pose[1]
    with np.errstate(invalid="ignore"):  # inf readings: inf - inf
        return c * dx + (-s) * dy, s * dx + c * dy


def angles(ch, angle_offset, angle_res, na):
    """win_angle of every angle of the search"""
    return [(ch - angle_offset) + float(np.uint32(k)) * angle_res for k in range(na)]


def exact_values(lx, ly, ch, angle_offset, angle_res, na, gox, goy, scale):
    """fp64 ((o + gox) - gox) * scale per axis [na][n] and their kround, as GridIndexLookup computes a lookup value
    (NaN for a non-finite point)"""
    vx, vy = np.empty((na, len(lx))), np.empty((na, len(lx)))
    with np.errstate(invalid="ignore"):
        for k, a in enumerate(angles(ch, angle_offset, angle_res, na)):
            c, s = math.cos(a), math.sin(a)
            ox, oy = c * lx - s * ly, s * lx + c * ly
            vx[k], vy[k] = ((ox + gox) - gox) * scale, ((oy + goy) - goy) * scale
    return vx, vy, kround(vx), kround(vy)


def _cos_sin_borderline(a):
    """(float)cos(a) or (float)sin(a) changes when the double moves by one unit in the last place"""
    out = False
    for v in (math.cos(a), math.sin(a)):
        for d in (-math.inf, math.inf):
            out |= f32(np.nextafter(v, d)) != f32(v)
    return bool(out)


class Brackets:
    """The fp32 brackets of every (group, beam): arrays [ng][n]"""

    def __init__(self, lx, ly, ch, angle_offset, angle_res, na, gox, goy, scale):
        n = len(lx)
        self.na, self.ng, self.n = na, (na + GROUP - 1) // GROUP, n
        ang = angles(ch, angle_offset, angle_res, na)
        cf = np.array([f32(math.cos(a)) for a in ang], dtype=f32)
        sf = np.array([f32(math.sin(a)) for a in ang], dtype=f32)
        px, py = np.asarray(lx).astype(f32), np.asarray(ly).astype(f32)
        scf = f32(scale)
        mg_match = f32(f32(4e-3) + f32(1e-15 * (abs(gox) + abs(goy)) * scale))
        with np.errstate(invalid="ignore", over="ignore"):
            mg = (mg_match + (f32(1e-5) * (np.abs(px) + np.abs(py))) * scf).astype(f32)
            # members k0 .. k0 + 3, the last group repeating its last angle as the kernel does
            ks = np.minimum(np.arange(self.ng)[:, None] * GROUP + np.arange(GROUP)[None, :], na - 1)  # [ng][4]
            x = (cf[ks][:, :, None] * px[None, None, :] - sf[ks][:, :, None] * py[None, None, :]).astype(f32)
            y = (sf[ks][:, :, None] * px[None, None, :] + cf[ks][:, :, None] * py[None, None, :]).astype(f32)
            self.xl = (x.min(axis=1) * scf - mg).astype(f32)
            self.xh = (x.max(axis=1) * scf + mg).astype(f32)
            self.yl = (y.min(axis=1) * scf - mg).astype(f32)
            self.yh = (y.max(axis=1) * scf + mg).astype(f32)
            ends = (self.xl, self.xh, self.yl, self.yh)
            self.inside = np.logical_and.reduce([np.abs(e) < f32(LIMIT) for e in ends])  # False for NaN too
            lo = lambda e: np.ceil((e - f32(0.5)).astype(f32))  # noqa: E731
            hi = lambda e: np.floor((e + f32(0.5)).astype(f32))  # noqa: E731
            self.mx, self.Mx = np.where(self.inside, lo(self.xl), 0).astype(np.int64), np.where(self.inside, hi(self.xh), 0).astype(np.int64)
            self.my, self.My = np.where(self.inside, lo(self.yl), 0).astype(np.int64), np.where(self.inside, hi(self.yh), 0).astype(np.int64)
            self.corner = self.inside & (self.Mx - self.mx <= SPREAD) & (self.My - self.my <= SPREAD)
            self.fallback = ~self.corner
            # distance of each end from the boundary its rounding (or the 8192 test) turns on
            d = []
            for e, sh in ((self.xl, -0.5), (self.xh, 0.5), (self.yl, -0.5), (self.yh, 0.5)):
                v = e.astype(np.float64) + sh
                d.append(np.minimum(np.abs(v - np.round(v)), np.abs(LIMIT - np.abs(e.astype(np.float64)))))
            self.edge = np.where(np.isfinite(px)[None, :] & np.isfinite(py)[None, :], np.min(d, axis=0), np.inf)
        trig = np.array([_cos_sin_borderline(a) for a in ang])
        self.trig_border = trig[ks].any(axis=1)  # [ng]
        self.borderline = (self.edge < BORDER) | self.trig_border[:, None]
        self.members = ks
        self.cnt = np.minimum(GROUP, na - np.arange(self.ng) * GROUP)

    def slack(self, vx, vy, finite):
        """the smallest distance (cells) by which a bracket that takes the corner, or is inside 8192, contains the
        unrounded exact values of its members, and whether every rounded exact value lies in [m, M]"""
        ok, worst = True, np.inf
        for j in range(GROUP):
            k = self.members[:, j]
            use = self.inside & finite[None, :]
            for lo_e, hi_e, m, M, v in ((self.xl, self.xh, self.mx, self.Mx, vx), (self.yl, self.yh, self.my, self.My, vy)):
                vk = v[k]
                s = np.minimum(vk - lo_e.astype(np.float64), hi_e.astype(np.float64) - vk)[use]
                if s.size:
                    worst = min(worst, float(s.min()))
                r = kround(vk)
                ok &= bool(((r >= m) & (r <= M))[use].all())
        return worst, ok

    def corner_class(self, base00, ws, lead, data_size):
        """[ng][n]: the low corner's flat index (int32 arithmetic) and class: 0 in the pooled planes, 4 read with the
        range test, 255 every corner outside; -1 where the beam takes the fallback"""
        a = ((base00 + self.mx + self.my * ws + 2**31) % 2**32) - 2**31
        last = a + 28 * ws + 28
        cls = np.where((last < -lead) | (a >= data_size), 255,
                       np.where((a >= -lead) & (last <= data_size + 4 * (32 - 8)), 0, 4))
        return a, np.where(self.corner, cls, -1)


def window_outside(a, ws, data_size):
    """win_origin_class's dropped test of a pruned sweep's window (32 rows, a 32-byte tile row, 8 bytes of alignment)"""
    ac = np.clip(a, -(1 << 29), 1 << 29)
    return (ac + min(SPAN * ws + 32 + 8, 1 << 29) < 0) | (ac - 8 >= data_size)


def group_bounds(grid, g, lut, base00, n, se, params, ch, br):
    """gub[g] of k_sweep_bound<., BOUND_GROUPS> from the brackets br (every beam, empty windows included)"""
    ws, ds = g.width_step, g.data_size
    nx, ny = _steps(se)
    P7, lead = pooled7(grid, ws), 8 * ws
    na, ng = lut.shape[0], br.ng

    def P7_at(f):
        f = ((f + 2**31) % 2**32) - 2**31
        return np.where((f >= -lead) & (f < ds), P7[np.clip(f + lead, 0, len(P7) - 1)], 0)

    a, cls = br.corner_class(base00, ws, lead, ds)
    ex = ((base00 + lut.astype(np.int64) + 2**31) % 2**32) - 2**31   # [na][n] the members' exact origins
    live = (lut != INVALID) & ~window_outside(ex, ws, ds)
    u = np.zeros((ng, 8, 8), dtype=np.int64)
    for by in range(8):
        for bx in range(8):
            off = 4 * by * ws + 4 * bx
            at_corner = np.where(cls == 255, 0, P7_at(a + off))
            mem = np.zeros((ng, br.n), dtype=np.int64)
            for j in range(GROUP):
                k = br.members[:, j]
                valid = (j < br.cnt)[:, None] & live[k]
                mem = np.maximum(mem, np.where(valid, P7_at(ex[k] + off), 0))
            u[:, by, bx] = np.where(br.corner, at_corner, mem).sum(axis=1)
    sums = np.repeat(np.repeat(u.transpose(1, 2, 0), 4, axis=0), 4, axis=1)[:ny, :nx]
    r = sums / float(n * 100)
    if se.do_penalize:
        pen = penalties(se, params, ch, nx, ny, na)
        r = r * np.stack([pen[:, :, h * GROUP:h * GROUP + GROUP].max(axis=2) for h in range(ng)], axis=2)
    return r.reshape(-1, ng).max(axis=0)


def _steps(se):
    from karto_volume_reference import abi
    return abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
