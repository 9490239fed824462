"""Float64 reference for ONE PL-ICP iteration — test code, nothing in the package imports it.

Written from the algorithm (A. Censi, "An ICP variant using a point-to-line metric", ICRA 2008) and the rules the
b2s_icp_params fields and the plicp.cu header name, not from oracle/plicp_oracle.c or the kernel:

  * LaserScanToLDP: a reading is valid iff range_min < r < range_max (NaN / inf / 0 / negative are not);
  * the current scan is moved by the running estimate x = (t, theta);
  * correspondence of a moved point p: the nearest valid reference point j1 within max_correspondence_dist among the
    beams of the angular window [floor(c - w), ceil(c + w)] clipped to [0, n - 1], where c = (atan2(p) - theta_0) /
    (theta_{n-1} - theta_0) * n (atan2 brought into [theta_0, theta_{n-1}] by +-2 pi where it falls outside),
    w = ceil((|max_angular_correction| + |atan(max_linear_correction / |p|)|) / ((theta_{n-1} - theta_0) / n));
    ties go to the lowest index; j1 = 0 or n - 1 is rejected; the segment end j2 is the nearer of the next valid
    reference beams above and below j1 (the lower one on a tie);
  * outliers_remove_doubles: of the points that chose the same j1, those farther than 3x the smallest squared
    distance to it are dropped;
  * trimming on the point-to-segment distance d (point-to-point: the distance to j1):
    keep d <= min(sort(d)[floor(k maxPerc)], mult * sort(d)[floor(k order)]), indices clipped to [0, k - 1];
  * fewer than 5 kept correspondences, or no finite solution, fails the iteration;
  * the point-to-line solve (GPC) minimises sum_i (R p_i + t - q_i)^T C_i (R p_i + t - q_i) with C_i = n_i n_i^T
    (n_i the unit normal of the segment j1 j2; C = I point to point).  Here it is solved NOT by the quartic of the
    Lagrange multiplier but by eliminating t (its optimum is linear for a fixed theta) and minimising the resulting
    one-dimensional function of theta: every stationary point is bracketed on a fine grid and located with brentq;
  * convergence: the increment expressed in the old pose's frame is below epsilon_xy in length and epsilon_theta in
    (wrapped) angle.

Every discrete decision the iteration takes is reported with its margin.  A step is *borderline* when one of them
lies within TOL (relative; for lengths with an absolute floor of LEN_TOL times the scene's size) of flipping: only then
may two correct implementations that round differently in the last place disagree on the correspondences.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
from scipy.optimize import brentq

TOL = 1e-9       # relative margin of a decision
LEN_TOL = 1e-12  # absolute floor for lengths, as a fraction of the scene's size: ~10^4 times the rounding of a coordinate
MIN_CORRESPONDENCES = 5


@dataclass
class Step:
    valid: int
    nvalid: int
    x: np.ndarray
    error: float
    converged: bool
    borderline: list = field(default_factory=list)  # names of the decisions that were within TOL of flipping
    j1: np.ndarray | None = None
    j2: np.ndarray | None = None
    kept: np.ndarray | None = None
    step_xy: float = np.nan  # length of the increment in the old pose's frame
    step_th: float = np.nan  # |wrapped angle| of the increment
    k: int = 0               # correspondences before trimming


def ldp(ranges, theta, range_min, range_max):
    r = np.asarray(ranges, np.float64)
    ok = (r > range_min) & (r < range_max)  # NaN compares false
    with np.errstate(invalid="ignore"):
        x = np.where(ok, r * np.cos(theta), 0.0)
        y = np.where(ok, r * np.sin(theta), 0.0)
    return ok, x, y


def _near_int(v, tol):
    return np.abs(v - np.round(v)) <= tol * np.maximum(1.0, np.abs(v))


def _window_cell(P, n, theta, wx, wy, st_raw):
    t0, t1 = theta[0], theta[-1]
    st = np.where(st_raw < t0, st_raw + 2 * np.pi, st_raw)
    st = np.where(st > t1, st - 2 * np.pi, st)
    return (st - t0) / (t1 - t0) * n


def _best_in(Drow, ok_row, lo, hi, max_d2):
    idx = np.arange(lo, hi + 1)
    d = Drow[lo:hi + 1]
    m = ok_row[lo:hi + 1] & (d <= max_d2)
    if not m.any():
        return -1
    return int(idx[m][np.argmin(d[m])])


def step(P, ref_ranges, sens_ranges, theta, range_min, range_max, x_old, tol=TOL, len_tol=LEN_TOL):
    """One iteration from the estimate x_old.  Returns a Step; on failure x is x_old."""
    theta = np.asarray(theta, np.float64)
    n = len(theta)
    x_old = np.asarray(x_old, np.float64)
    rv, rx, ry = ldp(ref_ranges, theta, range_min, range_max)
    sv, sx, sy = ldp(sens_ranges, theta, range_min, range_max)
    pts = np.concatenate([np.abs(rx[rv]), np.abs(ry[rv]), np.abs(sx[sv]), np.abs(sy[sv]), [1.0]])
    scale = pts.max() + np.abs(x_old[:2]).max()
    tl = len_tol * scale  # a length difference below this may be rounding in the coordinates
    flags = []

    c, s = np.cos(x_old[2]), np.sin(x_old[2])
    wx, wy = c * sx - s * sy + x_old[0], s * sx + c * sy + x_old[1]

    # ---- angular window
    t0, t1 = theta[0], theta[-1]
    ang_res = (t1 - t0) / n
    with np.errstate(divide="ignore"):
        nrm = np.hypot(wx, wy)
        q = (abs(np.deg2rad(P.max_angular_correction_deg)) + np.abs(np.arctan(P.max_linear_correction / nrm))) / ang_res
    w = np.ceil(q)
    st_raw = np.arctan2(wy, wx)
    cell = _window_cell(P, n, theta, wx, wy, st_raw)
    frm = np.clip(np.floor(cell - w), 0, n - 1).astype(np.int64)
    to = np.clip(np.ceil(cell + w), 0, n - 1).astype(np.int64)
    amb_win = sv & (_near_int(q, tol) | _near_int(cell - w, tol) | _near_int(cell + w, tol)
                    | (np.abs(st_raw - t0) <= tol * np.pi) | (np.abs(st_raw - t1) <= tol * np.pi))

    # ---- nearest valid reference point in the window, within max_correspondence_dist
    D = (wx[:, None] - rx[None, :]) ** 2 + (wy[:, None] - ry[None, :]) ** 2
    cols = np.arange(n)[None, :]
    inwin = (cols >= frm[:, None]) & (cols <= to[:, None]) & rv[None, :] & sv[:, None]
    max_d2 = P.max_correspondence_dist * P.max_correspondence_dist
    cand = inwin & (D <= max_d2)
    Dm = np.where(cand, D, np.inf)
    best = np.argmin(Dm, axis=1)
    rows = np.arange(n)
    bd = Dm[rows, best]
    best = np.where(np.isfinite(bd), best, -1)
    has = best >= 0
    # margins: a near-tie with another (not coincident) reference point, a candidate at the distance cut-off
    bsafe = np.where(has, best, 0)
    coincident = (rx[None, :] == rx[bsafe][:, None]) & (ry[None, :] == ry[bsafe][:, None])
    second = np.where(coincident, np.inf, Dm).min(axis=1)
    sq_bd, sq_2 = np.sqrt(np.where(has, bd, np.inf)), np.sqrt(second)
    if np.any(has & np.isfinite(second) & (sq_2 - np.where(has, sq_bd, 0.0) <= tl)):
        flags.append("nearest-neighbour tie")
    sqD = np.sqrt(D)
    at_cut = inwin & (np.abs(sqD - P.max_correspondence_dist) <= tl) & (sqD <= sq_bd[:, None] + tl)
    if at_cut.any():
        flags.append("max_correspondence_dist")
    for i in np.nonzero(amb_win)[0]:  # re-run the search over every window the rounding could have produced
        outs = set()
        for sr in (st_raw[i] - tol * np.pi, st_raw[i] + tol * np.pi):
            ci = _window_cell(P, n, theta, wx[i], wy[i], sr)
            for wi in {np.ceil(q[i] * (1 - tol)), np.ceil(q[i] * (1 + tol))}:
                lo, hi = ci - wi, ci + wi
                for f in {np.floor(lo - tol * max(1, abs(lo))), np.floor(lo + tol * max(1, abs(lo)))}:
                    for t in {np.ceil(hi - tol * max(1, abs(hi))), np.ceil(hi + tol * max(1, abs(hi)))}:
                        outs.add(_best_in(D[i], rv, int(np.clip(f, 0, n - 1)), int(np.clip(t, 0, n - 1)), max_d2))
        outs = {-1 if o in (0, n - 1) else o for o in outs}  # an extremal choice is rejected below either way
        if outs != {-1 if best[i] in (0, n - 1) else int(best[i])}:
            flags.append("angular window edge")
            break

    # ---- extremal reference beams rejected; the segment end is the nearer valid index-neighbour
    best = np.where((best == 0) | (best == n - 1), -1, best)
    idx = np.arange(n)
    up_of = np.minimum.accumulate(np.where(rv, idx, n)[::-1])[::-1]  # first valid index >= j
    dn_of = np.maximum.accumulate(np.where(rv, idx, -1))               # last valid index <= j
    up = np.where(best >= 0, np.append(up_of[1:], n)[np.maximum(best, 0)], n)
    dn = np.where(best >= 0, np.insert(dn_of[:-1], 0, -1)[np.maximum(best, 0)], -1)
    up = np.where(up >= n, -1, up)
    best = np.where((best >= 0) & (up < 0) & (dn < 0), -1, best)
    du = (wx - rx[np.maximum(up, 0)]) ** 2 + (wy - ry[np.maximum(up, 0)]) ** 2
    dd = (wx - rx[np.maximum(dn, 0)]) ** 2 + (wy - ry[np.maximum(dn, 0)]) ** 2
    other = np.where(up < 0, dn, np.where(dn < 0, up, np.where(du < dd, up, dn)))
    both = (best >= 0) & (up >= 0) & (dn >= 0)
    same_pt = (rx[np.maximum(up, 0)] == rx[np.maximum(dn, 0)]) & (ry[np.maximum(up, 0)] == ry[np.maximum(dn, 0)])
    if np.any(both & ~same_pt & (np.abs(np.sqrt(du) - np.sqrt(dd)) <= tl)):
        flags.append("segment end tie")
    j1, j2 = best, np.where(best >= 0, other, -1)
    use = j1 >= 0
    d2 = np.where(use, bd, 0.0)

    # ---- duplicate correspondences: keep those within 3x the best squared distance to the same reference point
    if P.outliers_remove_doubles:
        dj = np.full(n, np.inf)
        np.minimum.at(dj, j1[use], d2[use])
        lim3 = 3.0 * dj[np.maximum(j1, 0)]
        if np.any(use & (d2 != dj[np.maximum(j1, 0)]) & (np.abs(np.sqrt(d2) - np.sqrt(lim3)) <= tl)):
            flags.append("duplicate 3x rule")
        use = use & ~(d2 > lim3)

    # ---- trimming on the point-to-segment (or point-to-point) distance
    a_x, a_y = rx[np.maximum(j1, 0)], ry[np.maximum(j1, 0)]
    e_x, e_y = rx[np.maximum(j2, 0)] - a_x, ry[np.maximum(j2, 0)] - a_y
    if P.use_point_to_line_distance:
        len2 = e_x * e_x + e_y * e_y
        with np.errstate(invalid="ignore", divide="ignore"):
            u = np.where(len2 > 0, ((wx - a_x) * e_x + (wy - a_y) * e_y) / len2, 0.0)
        u = np.clip(u, 0.0, 1.0)
        dist = np.hypot(a_x + u * e_x - wx, a_y + u * e_y - wy)
    else:
        dist = np.sqrt(d2)
    k = int(use.sum())
    if k > 0:
        srt = np.sort(dist[use])
        o1 = min(max(int(np.floor(k * P.outliers_maxPerc)), 0), k - 1)
        o2 = min(max(int(np.floor(k * P.outliers_adaptive_order)), 0), k - 1)
        lim = min(srt[o1], P.outliers_adaptive_mult * srt[o2])
        gap = np.abs(dist - lim)
        if np.any(use & (gap > 0) & (gap <= max(tl, tol * lim))):
            flags.append("trimming limit")
        use = use & (dist <= lim)
    nvalid = int(use.sum())
    error = float(dist[use].sum())
    fail = Step(0, nvalid, x_old.copy(), error, False, flags, j1, j2, use, k=k)
    if nvalid < MIN_CORRESPONDENCES:
        return fail

    # ---- the point-to-line solve, by elimination of t and a 1-D search over theta
    i = np.nonzero(use)[0]
    px, py, qx, qy = sx[i], sy[i], rx[j1[i]], ry[j1[i]]
    if P.use_point_to_line_distance:
        nx, ny = ry[j1[i]] - ry[j2[i]], -(rx[j1[i]] - rx[j2[i]])
        with np.errstate(invalid="ignore", divide="ignore"):
            ln = np.hypot(nx, ny)
            nx, ny = nx / ln, ny / ln
        C = np.stack([np.stack([nx * nx, nx * ny], -1), np.stack([nx * ny, ny * ny], -1)], -2)
    else:
        C = np.broadcast_to(np.eye(2), (len(i), 2, 2))
    if not np.all(np.isfinite(C)):
        return fail
    a = np.stack([px, py], -1)
    b = np.stack([-py, px], -1)  # d/dtheta of R p at theta = 0, i.e. J p
    d = -np.stack([qx, qy], -1)
    Ca, Cb, Cd = (np.einsum("kij,kj->ki", C, v) for v in (a, b, d))
    X, Y, Z = np.sum(a * Ca), np.sum(b * Cb), np.sum(a * Cb)
    U, V, W = np.sum(a * Cd), np.sum(b * Cd), np.sum(d * Cd)
    A = C.sum(0)
    sa, sb, sd = Ca.sum(0), Cb.sum(0), Cd.sum(0)
    if np.linalg.det(A) == 0.0:
        return fail
    Ai = np.linalg.inv(A)

    def bvec(th):
        return np.cos(th) * sa + np.sin(th) * sb + sd

    def f(th):
        cc, ss = np.cos(th), np.sin(th)
        bb = bvec(th)
        return cc * cc * X + ss * ss * Y + 2 * cc * ss * Z + 2 * cc * U + 2 * ss * V + W - bb @ Ai @ bb

    def fp(th):
        cc, ss = np.cos(th), np.sin(th)
        bb, db = bvec(th), -ss * sa + cc * sb
        return 2 * cc * ss * (Y - X) + 2 * (cc * cc - ss * ss) * Z - 2 * ss * U + 2 * cc * V - 2 * (bb @ Ai @ db)

    grid = np.linspace(-np.pi, np.pi, 4097)
    g = np.array([fp(t) for t in grid])
    roots = []
    for k_ in range(len(grid) - 1):
        if g[k_] == 0.0:
            roots.append(grid[k_])
        elif g[k_] < 0.0 < g[k_ + 1]:
            roots.append(brentq(fp, grid[k_], grid[k_ + 1], xtol=1e-300, rtol=4 * np.finfo(float).eps, maxiter=400))
    if not roots:
        return fail
    th = min(roots, key=f)
    th = float(np.arctan2(np.sin(th), np.cos(th)))
    t = -Ai @ bvec(th)
    x_new = np.array([t[0], t[1], th])
    if not np.all(np.isfinite(x_new)):
        return fail

    # ---- convergence: the increment in the old pose's frame
    ddx, ddy = x_new[0] - x_old[0], x_new[1] - x_old[1]
    lx, ly = c * ddx + s * ddy, -s * ddx + c * ddy
    dth = (x_new[2] - x_old[2] + np.pi) % (2 * np.pi) - np.pi
    step_xy, step_th = float(np.hypot(lx, ly)), abs(float(dth))
    converged = step_xy < P.epsilon_xy and step_th < P.epsilon_theta
    return Step(1, nvalid, x_new, error, converged, flags, j1, j2, use, step_xy, step_th, k)


def iterate(P, ref_ranges, sens_ranges, theta, range_min, range_max, x0, xtol, tol=TOL):
    """Run step() until it fails, converges or reaches P.max_iterations, from x0.  Returns
    (valid, iterations, nvalid, x, borderline) where borderline names what came within TOL (or, for the convergence
    test, within xtol — the accuracy two solvers' estimates can be trusted to — and with xtol as the length floor,
    since two estimates xtol apart move every point by up to that much) of another outcome."""
    x = np.asarray(x0, np.float64).copy()
    flags, nvalid = [], 0
    for it in range(P.max_iterations):
        st = step(P, ref_ranges, sens_ranges, theta, range_min, range_max, x, tol, max(LEN_TOL, xtol))
        flags += st.borderline
        if not st.valid:
            return 0, it, st.nvalid, x, flags
        if min(abs(st.step_xy - P.epsilon_xy), abs(st.step_th - P.epsilon_theta)) <= xtol:
            flags.append("convergence test")
        x, nvalid = st.x, st.nvalid
        if st.converged:
            return 1, it + 1, nvalid, x, flags
    return 1, P.max_iterations, nvalid, x, flags
