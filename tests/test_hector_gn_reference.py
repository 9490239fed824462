"""The float64 Gauss-Newton reference (tests/hector_gn_reference.py) against the float32 restatement
(PortHectorProcessor, pinned to the unmodified lesson4 headers), before any device path is held to it.

Every geometry of tests/hector_cases.py, families walk, long and interp_edge: the maps are the restatement's after a
mapping-only warm-up, the gate stays shut (min_dist = min_angle = 1e9), every scan is matched from its hint.

The Hessian bound.  The last H of a match is evaluated at the map pose before the final step; the float32 H is compared
with the float64 sums at the map pose recovered from the returned world pose, on converged scans only (the float64
match's last level-0 step below 1e-6 cells / rad).  The bound of each of the six distinct entries is
K * sum|term| + floor + pose_slack.  The floor is the absolute error of a float32 gradient (2^-22) times the other
factor of each term: a gradient near zero has no relative accuracy.  pose_slack covers the rounding of the recovered pose: its smooth part (about 3e-5 of
sum|term| on these cases) and the points within that rounding of a cell edge, whose gradient jumps (rare, but up to
6e-3 of sum|term| on a scan where one lands).  Without that slack, one such point per ~10 scans breaks any bound near
the float32 summation rounding (raw |H32 - H64| / sum|term| reached 3.5e-3 on a converged scan).

K = 1e-5.  A float32 sum of n terms carries a rounding of order sqrt(n) * 2^-24 * sum|term| (about 3e-6 at 2048
terms); the largest excess observed here over floor and slack, on the 78 converged walk and long scans of 575 points
or more (of 132) and the converged interp_edge scans, is 4.0e-6 of sum|term| (wide, long, 2047 points).  A share or chunk boundary that drops or double-counts one point moves an entry by about 1/n of
sum|term|: 5e-4 at 2048 points, fifty times K."""
import numpy as np
import pytest

import hector_cases as hc
import hector_gn_reference as gr

FAMILIES = ("walk", "long", "interp_edge")


@pytest.fixture(scope="module")
def cases():
    return {(g, f): gr.cpu_case(g, f) for g in hc.GEOMETRIES for f in FAMILIES}


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_restatement_within_float64_bound(cases, geometry, family):
    c = cases[(geometry, family)]
    assert not c.flags.any()  # the gate stayed shut: every scan was matched against the warm-up maps
    for i, pts in enumerate(c.stream.scans):
        m = c.matches[i]
        r = gr.check_hessian(c, i, c.covs[i], c.poses[i])
        assert r is None or r <= gr.K, (i, len(pts), r)
        if len(pts) >= gr.MIN_POSE_POINTS and not m.singular:
            assert gr.pose_error(c.poses[i], m.pose) <= 1e-4, (i, c.poses[i], m.pose)
        if family == "interp_edge" and not m.singular:
            # NaN placement: a step through a singular H is rounding noise in either precision, elsewhere both agree
            assert np.isnan(c.poses[i]).any() == np.isnan(m.pose).any(), (i, c.poses[i], m.pose)


def test_most_long_scans_converge(cases):
    """The Hessian check must not be vacuous: most walk and long scans of 575 points or more converge, on every
    geometry with a map large enough to hold them (the 12 x 12 map matches nothing: every H is zero there)."""
    conv = tot = 0
    for (g, f), c in cases.items():
        if f == "interp_edge" or g == "tiny":
            continue
        for i, pts in enumerate(c.stream.scans):
            if len(pts) >= gr.MIN_POSE_POINTS:
                tot += 1
                conv += gr.converged(c.matches[i])
    assert conv >= tot // 2, (conv, tot)
    tiny = cases[("tiny", "walk")]
    assert all(not c.any() for c in tiny.covs)


def test_bound_sees_one_point():
    """Dropping one point of a 2048-point scan, or counting one twice, moves some H entry beyond the bound at the same
    pose (no slack: the pose is exact), on every geometry whose map sees the scan, for any point of at least average
    weight in some entry (a point in a flat part of the map adds next to nothing: no bound can see it)."""
    for g in hc.GEOMETRIES:
        if g == "tiny":
            continue
        c = gr.cpu_case(g, "long")
        pts, hint = c.stream.scans[-1], c.stream.hints[-1]
        lvl = c.levels[0]
        mp = lvl.map_coords32(hint)
        full = gr.hessian_at(lvl, pts, mp)
        d, h = gr.point_terms(lvl, mp, pts)
        weight = (np.abs(h) / np.abs(h).sum(1, keepdims=True)).max(0)
        seen = np.flatnonzero(weight >= 1.0 / len(pts))
        assert len(seen) > len(pts) // 20, (g, len(seen))
        for j in (seen[len(seen) // 4], seen[len(seen) // 2], seen[-1]):  # three points spread over the scan
            for sign in (-1.0, 1.0):
                H = full.H + sign * gr._sym(h[:, j])
                assert gr.hessian_excess(H, full) > gr.K, (g, j, sign)
