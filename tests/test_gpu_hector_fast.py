"""GPU tests of the Hector processor's fast mode (set_exact(0)) against the float64 Gauss-Newton reference
(tests/hector_gn_reference.py, itself checked against the restatement by tests/test_hector_gn_reference.py), on every
geometry of tests/hector_cases.py, families walk, long (1 ... 2048 points: the 4-CTA shares around 576, 1152 and 2048)
and interp_edge.  Its three match paths:
- one CTA, hs_match_cta<false, false> (B2S_HS_CLUSTER=0 when the handle is created);
- the 4-CTA cluster, k_hs_stream<false, true>: the master sums the helpers' shares (hs_share, hs_match_helper);
- the fleet, k_hs_stream_batch<false>: process_stream_batch, the three families as three processors of one handle.
The exact path runs beside them as the control: it meets the same bound.

Per scan: the last Hessian within K * sum|term| + pose_slack of the float64 sums at the returned pose (converged scans),
the pose within 1e-4 of the restatement (575 points or more), the same (shut) gate decision.  Then the single-map
handle's match (k_hc_match, hector_map.cu) across its 1024-point staging chunks, on the non-square geometries."""
import numpy as np
import pytest

import hector_cases as hc
import hector_gn_reference as gr
from oracle import port

pytestmark = pytest.mark.gpu
FAMILIES = ("walk", "long", "interp_edge")


@pytest.fixture(scope="module")
def H(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector")


@pytest.fixture(scope="module")
def cases():
    return {}


def _case(cases, geometry, family):
    if (geometry, family) not in cases:
        cases[(geometry, family)] = gr.cpu_case(geometry, family)
    return cases[(geometry, family)]


def _levels_equal(g, c_levels_of, levels, what, b=None):
    for lvl in range(levels):
        got = g.level(lvl) if b is None else g.level_of(b, lvl)
        bad, touched = hc.cell_mismatch(got, c_levels_of(lvl))
        assert bad == 0, (what, lvl, bad, touched)


def _restatement_maps(case, family):
    c = port.PortHectorProcessor(**case.kw)
    gr.warm_up(c, case.stream, family)
    return c


def _check_scan(case, i, pose, cov, flag, what):
    """One device scan against the float64 reference and the restatement.  Returns whether the Hessian was checked."""
    pts = case.stream.scans[i]
    assert flag == case.flags[i], (what, i)
    r = gr.check_hessian(case, i, cov, pose)
    assert r is None or r <= gr.K, (what, i, len(pts), r)
    if len(pts) >= gr.MIN_POSE_POINTS:
        assert gr.pose_error(pose, case.poses[i]) <= 1e-4, (what, i, pose, case.poses[i])
    return r is not None


def _single_handle_run(H, case, family, exact):
    g = H.HectorSlam(exact=exact, **case.kw)
    gr.warm_up(g, case.stream, family)
    c = _restatement_maps(case, family)
    _levels_equal(g, c.level, case.kw["levels"], ("warm-up", exact))  # the mapping is exact in both modes
    c.close()
    out = [g.update(pts, (0, 0), case.stream.hints[i]) + (g.map_updated,) for i, pts in enumerate(case.stream.scans)]
    return g, out


@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_single_stream_fast_paths(H, cases, geometry, monkeypatch):
    """One-CTA fast, clustered fast (where cluster launches exist) and the exact control, scan by scan (update())."""
    checked = 0
    for family in FAMILIES:
        case = _case(cases, geometry, family)
        runs = {}
        monkeypatch.setenv("B2S_HS_CLUSTER", "0")
        runs["one-cta"] = _single_handle_run(H, case, family, False)
        monkeypatch.delenv("B2S_HS_CLUSTER")
        assert runs["one-cta"][0].cluster_size() == 1
        runs["exact"] = _single_handle_run(H, case, family, True)
        g, out = _single_handle_run(H, case, family, False)
        if g.cluster_size() == 4:  # (a cluster exchange that timed out fails update() itself)
            runs["cluster"] = (g, out)
        for what, (g, out) in runs.items():
            for i, (pose, cov, flag) in enumerate(out):
                checked += _check_scan(case, i, pose, cov, flag, (geometry, family, what))
                if what == "exact":
                    assert hc.same_bits(pose, case.poses[i]) and hc.same_bits(cov, case.covs[i]), (family, i)
            g.close()
    assert checked > 0 or geometry == "tiny"


@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_fleet_fast(H, cases, geometry):
    """process_stream_batch in fast mode (k_hs_stream_batch<false>): the three families as three processors of one
    handle, warmed up and then stepped one scan per call (a processor whose stream has ended gets none), so that every
    scan's Hessian comes back."""
    fam_cases = [_case(cases, geometry, f) for f in FAMILIES]
    kw = fam_cases[0].kw
    B = len(FAMILIES)
    g = H.HectorSlam(batch=B, max_points=2048, exact=False, **kw)
    warm = [gr.warm_scans(c.stream, f) for c, f in zip(fam_cases, FAMILIES)]
    for i in range(4):
        step = [[w[0][i]] for w in warm]
        hints = [w[1][i:i + 1] for w in warm]
        g.process_stream_batch(step, (0, 0), pose_hints=hints)
        g.process_stream_batch(step, (0, 0), pose_hints=hints, map_without_matching=True)
    for b, (c, f) in enumerate(zip(fam_cases, FAMILIES)):
        r = _restatement_maps(c, f)
        _levels_equal(g, r.level, kw["levels"], ("fleet warm-up", f), b=b)
        r.close()
    for i in range(max(len(c.stream) for c in fam_cases)):
        live = [i < len(c.stream) for c in fam_cases]
        step = [[c.stream.scans[i]] if ok else [] for c, ok in zip(fam_cases, live)]
        hints = [c.stream.hints[i:i + 1] if ok else np.zeros((0, 3), np.float32) for c, ok in zip(fam_cases, live)]
        res, covs = g.process_stream_batch(step, (0, 0), pose_hints=hints)
        for b, (c, ok) in enumerate(zip(fam_cases, live)):
            if ok:
                _check_scan(c, i, res[b][0][0], covs[b], res[b][1][0], (geometry, FAMILIES[b], "fleet"))
    g.close()


# (deep: the 8-level processor loses the self-driven walk in the restatement itself, jumping metres between scans, so
# its gate decisions there hinge on the last bit of a pose)
@pytest.mark.parametrize("geometry", [g for g in hc.GEOMETRIES if g != "deep"])
def test_self_driven_cells(H, geometry, monkeypatch):
    """The walk self-driven (each hint the previous match) with the gate open, one-CTA and clustered fast mode: the
    same gate decisions as the restatement and cells within the fast mode's touched // 500.  (Poses are not held to
    1e-4 here: that contract is per match from the same hint, and a self-driven stream compounds it.)"""
    kw = hc.processor_kw(geometry)
    s = hc.make_stream(geometry, "walk")
    c = port.PortHectorProcessor(**kw)
    _, _, fc = hc.run_stream(c, s, "self")
    monkeypatch.setenv("B2S_HS_CLUSTER", "0")
    g1 = H.HectorSlam(exact=False, **kw)
    monkeypatch.delenv("B2S_HS_CLUSTER")
    gc = H.HectorSlam(exact=False, **kw)
    for g in (g1, gc) if gc.cluster_size() == 4 else (g1,):
        _, ug, _ = g.process_stream(s.scans, (0, 0), first_hint=s.first)
        assert np.array_equal(ug, fc), (geometry, ug, fc)
        for lvl in range(kw["levels"]):
            bad, touched = hc.cell_mismatch(g.level(lvl), c.level(lvl))
            assert bad <= max(2, touched // 500), (geometry, lvl, bad, touched)
        g.close()
    c.close()


CHUNK_LENGTHS = (1, 1023, 1024, 1025, 2048, 2049, 3073)


def _single_maps(H, geometry):
    gm = hc.GEOMETRIES[geometry]
    sx, sy, res, (stx, sty) = gm["size_x"], gm["size_y"], gm["resolution"], gm["start"]
    s = hc.make_stream(geometry, "walk")
    g, c = H.HectorMap(sx, sy, res, stx, sty), port.PortHectorMap(sx, sy, res, stx, sty)
    g.set_factors(0.4, 0.9), c.set_factors(0.4, 0.9)
    longs = hc.make_stream(geometry, "batch_long")
    for i in range(len(s)):
        g.update_by_scan(s.scans[i], (0, 0), s.hints[i])
        c.update_by_scan(s.scans[i], (0, 0), s.hints[i])
    for i in range(len(longs)):
        g.update_by_scan(longs.scans[i], (0, 0), longs.hints[i])
        c.update_by_scan(longs.scans[i], (0, 0), longs.hints[i])
    assert hc.cell_mismatch(g.cells(), c.cells())[0] == 0
    level = gr.make_level(c.cells()[0], res, sx, sy, (stx, sty), 0)
    return g, c, level, longs


@pytest.mark.parametrize("geometry", ["wide", "tall_odd", "edge"])
def test_single_map_chunks(H, geometry):
    """b2s_hector_map_match_data across the 1024-point staging chunks of k_hc_match.  max_iterations = 0: H is evaluated
    exactly at the begin pose (its float32 map pose is reproducible), so it meets K * sum|term| with no pose slack;
    the device's expf probabilities differ from the double exp in the last bit, inside K.  max_iterations = 5: the
    pose within 1e-4 of the restatement."""
    g, c, level, longs = _single_maps(H, geometry)
    src = longs.scans[-1]  # 4096 points
    begin = (longs.hints[-1] + np.array([0.02, -0.015, 0.01], np.float32)).astype(np.float32)
    mp = level.map_coords32(begin)
    for n in CHUNK_LENGTHS:
        pts = np.ascontiguousarray(src[:n])
        eg, Hg = g.match_data(pts, begin, 0)
        sums = gr.hessian_at(level, pts, mp)
        r = gr.hessian_excess(Hg, sums)
        assert r <= gr.K, (geometry, n, r)
        if n >= gr.MIN_POSE_POINTS:
            ec, _ = c.match_data(pts, begin, 0)
            assert gr.pose_error(eg, ec) <= 1e-4, (geometry, n, eg, ec)
            eg, _ = g.match_data(pts, begin, 5)
            ec, _ = c.match_data(pts, begin, 5)
            assert gr.pose_error(eg, ec) <= 1e-4, (geometry, n, eg, ec)
    g.close(), c.close()


@pytest.mark.parametrize("geometry", ["wide", "tall_odd", "edge"])
def test_single_map_no_point_inside(H, geometry):
    """Every point outside the map: H[0] == 0, so no step is taken.  The pose comes back as the begin pose through
    the map transform and normalize_angle (bit for bit the restatement's) and H is zero, at any chunk count."""
    g, c, level, longs = _single_maps(H, geometry)
    sx = hc.GEOMETRIES[geometry]["size_x"]
    begin = (longs.hints[-1] + np.array([0.0, 0.0, 2 * np.pi], np.float32)).astype(np.float32)
    for n in (1, 1024, 2049):
        pts = np.ascontiguousarray(longs.scans[-1][:n] + np.float32(4 * sx))
        eg, Hg = g.match_data(pts, begin, 5)
        ec, Hc = c.match_data(pts, begin, 5)
        assert not Hg.any() and not Hc.any(), (geometry, n)
        assert hc.same_bits(eg, ec), (geometry, n, eg, ec)
        assert gr.pose_error(eg, begin) <= 1e-5 and -np.pi < eg[2] <= np.pi, (geometry, n, eg, begin)
    g.close(), c.close()
