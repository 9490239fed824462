"""GPU tests of the batched stream call (b2s_hector_slam_process_stream_batch, k_hs_stream_batch): every processor of a
handle walks its own recording in one launch, one CTA per processor.

Each processor's poses, gate decisions, last Hessian, last poses and every cell of every level must equal the
restatement (PortHectorProcessor, pinned to the unmodified lesson4 headers by tests/test_hector_edges_reference.py) run
over that processor's scans alone, bit for bit in exact mode; and equal the per-step batch path (update_batch) fed the
same streams, in both modes."""
import ctypes as C

import numpy as np
import pytest

import hector_cases as hc
from oracle import port

pytestmark = pytest.mark.gpu
FLT_MAX = np.float32(3.402823466e+38)  # HectorSlamProcessor::reset's last map-update pose


@pytest.fixture(scope="module")
def H(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector")


def _no_scans(first):
    return hc.Stream([], np.zeros((0, 3), np.float32), np.asarray(first, np.float32))


def _sub(s, lo, hi):
    return hc.Stream(s.scans[lo:hi], s.hints[lo:hi], s.hints[lo] if lo > 0 else s.first)


def _ragged_fleet():
    """Wide map, seven processors: no scans, one scan, only empty scans, the long family (1 ... 2048 points), the
    batch_long family (2049 ... 4096), the wide walk and the edge map's walk."""
    walk, edge = hc.make_stream("wide", "walk"), hc.make_stream("edge", "walk")
    empties = hc.Stream([np.zeros((0, 2), np.float32)] * 3, walk.hints[:3], walk.first)
    return [_no_scans(walk.first), _sub(walk, 0, 1), empties, hc.make_stream("wide", "long"),
            hc.make_stream("wide", "batch_long"), walk, edge]


def _fleet_call(g, procs, form, origo=(0, 0)):
    streams = [p.scans for p in procs]
    if form == "self":
        return g.process_stream_batch(streams, origo, first_hints=np.stack([p.first for p in procs]))
    return g.process_stream_batch(streams, origo, pose_hints=[p.hints for p in procs], map_without_matching=form == "given")


def _cpu(kw, s, form, origo=(0, 0)):
    """The restatement over one processor's scans: (processor, poses [n, 3], flags [n], last covariance)."""
    c = port.PortHectorProcessor(**kw)
    est, poses, flags, cov = s.first, [], [], None
    for i, pts in enumerate(s.scans):
        est, cov = c.update(pts, origo, est if form == "self" else s.hints[i], form == "given")
        poses.append(np.asarray(est, np.float32)), flags.append(c.map_updated)
    return c, np.array(poses, np.float32).reshape(-1, 3), np.array(flags, bool), cov


def _last_update_pose(poses, flags):
    return poses[np.flatnonzero(flags)[-1]] if flags.any() else np.full(3, FLT_MAX, np.float32)


def _levels_equal(g, b, c, levels, what):
    for lvl in range(levels):
        bad, touched = hc.cell_mismatch(g.level_of(b, lvl), c.level(lvl))
        assert bad == 0, (what, lvl, bad, touched)


def _check_fleet(g, procs, res, covs, kw, form, what):
    """Every processor of a fleet call against the restatement over its own scans."""
    for b, s in enumerate(procs):
        c, pc, fc, cc = _cpu(kw, s, form)
        pg, fg = res[b]
        assert hc.same_bits(pg, pc), (what, form, b, np.flatnonzero(~((pg == pc) | (np.isnan(pg) & np.isnan(pc))).all(1)))
        assert np.array_equal(fg, fc), (what, form, b, fg, fc)
        if len(s) and form != "given":
            assert hc.same_bits(covs[b], cc), (what, form, b)
        else:  # untouched row
            assert not covs[b].any(), (what, form, b)
        a, u = g.last_poses(b)
        if len(s):
            assert hc.same_bits(a, pc[-1]) and hc.same_bits(u, _last_update_pose(pc, fc)), (what, form, b)
        _levels_equal(g, b, c, kw["levels"], (what, form, b))
        c.close()


def test_ragged_fleet_exact(H):
    """Ragged recordings on one max_points = 4096 handle, self-driven, with hints and mapping only, against the
    restatement; processors whose scans fit 2048 points also against a single handle's process_stream."""
    kw = hc.processor_kw("wide")
    procs = _ragged_fleet()
    for form in ("self", "hints", "given"):
        g = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
        res, covs = _fleet_call(g, procs, form)
        _check_fleet(g, procs, res, covs, kw, form, "ragged")
        for b, s in enumerate(procs):
            if b == 4 or not len(s):  # (batch_long exceeds the single handle; an empty stream is a no-op there)
                continue
            g1 = H.HectorSlam(**kw)
            if form == "self":
                p1, u1, c1 = g1.process_stream(s.scans, (0, 0), first_hint=s.first)
            else:
                p1, u1, c1 = g1.process_stream(s.scans, (0, 0), pose_hints=s.hints, map_without_matching=form == "given")
            assert hc.same_bits(res[b][0], p1) and np.array_equal(res[b][1], u1), (form, b)
            if form != "given":
                assert hc.same_bits(covs[b], c1), (form, b)
            for lvl in range(kw["levels"]):
                assert hc.cell_mismatch(g.level_of(b, lvl), g1.level(lvl))[0] == 0, (form, b, lvl)
            g1.close()
        g.close()


def test_single_processor_handle(H):
    """B = 1 (b2s_hector_slam_create): the batched call equals process_stream on a twin handle."""
    kw = hc.processor_kw("wide")
    s = hc.make_stream("wide", "empty")
    ga, gb = H.HectorSlam(**kw), H.HectorSlam(**kw)
    res, covs = ga.process_stream_batch([s.scans], (0, 0), first_hints=s.first[None])
    p1, u1, c1 = gb.process_stream(s.scans, (0, 0), first_hint=s.first)
    assert hc.same_bits(res[0][0], p1) and np.array_equal(res[0][1], u1) and hc.same_bits(covs[0], c1)
    for lvl in range(kw["levels"]):
        assert hc.cell_mismatch(ga.level(lvl), gb.level(lvl))[0] == 0, lvl


@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_every_geometry(H, geometry):
    """Three processors (walk, walk with empty scans, interpolation-limit scans) on every geometry of hector_cases:
    non-square both ways, a robot near two edges, 1 / 4 / 8 levels, 12 x 12."""
    kw = hc.processor_kw(geometry)
    procs = [hc.make_stream(geometry, f) for f in ("walk", "empty", "interp_edge")]
    for form in ("self", "hints", "given"):
        g = H.HectorSlam(batch=3, max_points=2048, **kw)
        res, covs = _fleet_call(g, procs, form)
        _check_fleet(g, procs, res, covs, kw, form, geometry)
        g.close()


def _equal_fleet():
    """Five processors of six scans each, on the wide map."""
    walk, edge, empty = hc.make_stream("wide", "walk"), hc.make_stream("edge", "walk"), hc.make_stream("wide", "empty")
    tall, longs = hc.make_stream("tall_odd", "walk"), hc.make_stream("wide", "long")
    return [_sub(walk, 0, 6), _sub(edge, 4, 10), _sub(empty, 0, 6), _sub(tall, 6, 12), _sub(longs, 13, 19)]


@pytest.mark.parametrize("exact", [True, False])
def test_equal_streams_equal_stepping(H, exact):
    """Equal-length recordings: the fleet call equals update_batch stepped scan by scan (first step with the first
    hints, then chained through each processor's last scan-match pose), bit for bit in both modes: both run
    hs_match_cta<EXACT, false> and the same mark / apply passes."""
    kw = hc.processor_kw("wide")
    procs = _equal_fleet()
    B, n = len(procs), len(procs[0])
    gf = H.HectorSlam(batch=B, max_points=2048, exact=exact, **kw)
    gs = H.HectorSlam(batch=B, max_points=2048, exact=exact, **kw)
    res, covs = _fleet_call(gf, procs, "self")
    for i in range(n):
        hints = np.stack([p.first for p in procs]) if i == 0 else None
        ps, cs, us = gs.update_batch([p.scans[i] for p in procs], (0, 0), hints)
        for b in range(B):
            assert hc.same_bits(res[b][0][i], ps[b]) and res[b][1][i] == us[b], (exact, i, b)
    for b in range(B):
        assert hc.same_bits(covs[b], cs[b]), (exact, b)
        for x, y in zip(gf.last_poses(b), gs.last_poses(b)):
            assert hc.same_bits(x, y), (exact, b)
        for lvl in range(kw["levels"]):
            assert hc.cell_mismatch(gf.level_of(b, lvl), gs.level_of(b, lvl))[0] == 0, (exact, b, lvl)
    if exact:
        _check_fleet(gf, procs, res, covs, kw, "self", "stepping")


def test_fast_fleet_within_contract(H):
    """Fast mode against the restatement: after a mapping-only call the gate stays shut, so every processor matches
    its scans against the same maps as the CPU; poses within 1e-4 for scans of 575 points or more (the existing rule:
    a few points give a near-singular Hessian, where the tree sum may take another path)."""
    kw = dict(hc.processor_kw("wide"), min_dist=1e9, min_angle=1e9)
    longs, walk = hc.make_stream("wide", "long"), hc.make_stream("wide", "walk")
    warm = _sub(walk, 0, 4)
    procs = [longs, walk]
    g = H.HectorSlam(batch=2, max_points=2048, exact=False, **kw)
    g.process_stream_batch([warm.scans, warm.scans], (0, 0), pose_hints=[warm.hints, warm.hints], map_without_matching=True)
    res, _ = g.process_stream_batch([p.scans for p in procs], (0, 0), pose_hints=[p.hints for p in procs])
    for b, s in enumerate(procs):
        c = port.PortHectorProcessor(**kw)
        for i in range(len(warm)):
            c.update(warm.scans[i], (0, 0), warm.hints[i], True)
        for i, pts in enumerate(s.scans):
            ec, _ = c.update(pts, (0, 0), s.hints[i])
            if len(pts) >= 575:
                assert np.abs(res[b][0][i] - ec).max() <= 1e-4, (b, i, res[b][0][i], ec)
        c.close()


def test_two_halves_equal_one_call(H):
    """State persists between calls: each recording cut at its middle and run in two calls (the second chained through
    the last scan-match pose) equals one call."""
    kw = hc.processor_kw("wide")
    procs = _ragged_fleet()
    one = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
    two = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
    r1, c1 = _fleet_call(one, procs, "self")
    cut = [(len(p) + 1) // 2 for p in procs]  # (a one-scan recording is all first half: the second call chains)
    ra, ca = two.process_stream_batch([p.scans[:k] for p, k in zip(procs, cut)], (0, 0),
                                      first_hints=np.stack([p.first for p in procs]))
    rb, cb = two.process_stream_batch([p.scans[k:] for p, k in zip(procs, cut)], (0, 0))
    for b, p in enumerate(procs):
        assert hc.same_bits(np.concatenate([ra[b][0], rb[b][0]]), r1[b][0]), b
        assert np.array_equal(np.concatenate([ra[b][1], rb[b][1]]), r1[b][1]), b
        assert hc.same_bits(cb[b] if len(p) - cut[b] else ca[b], c1[b]), b
        for x, y in zip(two.last_poses(b), one.last_poses(b)):
            assert hc.same_bits(x, y), b
        for lvl in range(kw["levels"]):
            assert hc.cell_mismatch(two.level_of(b, lvl), one.level_of(b, lvl))[0] == 0, (b, lvl)


def test_more_processors_than_one_wave(H):
    """B = 300 on small maps (more CTAs than the device holds at once): every processor against the restatement."""
    kw = dict(size_x=96, size_y=80, resolution=0.05, start=(0.5, 0.5), levels=3, **hc.GATE)
    pool = [hc.make_stream(g, "walk") for g in ("wide", "edge", "tall_odd")]
    procs = []
    for b in range(300):
        s = pool[b % 3]
        k = 0 if b % 7 == 0 else 1 + b % 5
        lo = (b // 3) % 8
        procs.append(_sub(s, lo, lo + k) if k else _no_scans(s.hints[lo]))
    for form in ("self", "hints"):
        g = H.HectorSlam(batch=300, max_points=2048, **kw)
        res, covs = _fleet_call(g, procs, form)
        _check_fleet(g, procs, res, covs, kw, form, "300")
        g.close()


def test_epoch_wrap_inside_a_call(H):
    """A call that crosses the 20-bit stamp epoch (debug_set_epoch((1 << 20) - 3)) equals the same call without."""
    kw = hc.processor_kw("wide")
    procs = _ragged_fleet()
    ga = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
    gw = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
    gw.debug_set_epoch((1 << 20) - 3)
    for form in ("given", "self"):
        ra, ca = _fleet_call(ga, procs, form)
        rw, cw = _fleet_call(gw, procs, form)
        for b in range(len(procs)):
            assert hc.same_bits(ra[b][0], rw[b][0]) and np.array_equal(ra[b][1], rw[b][1]), (form, b)
        assert hc.same_bits(ca, cw), form
    for b in range(len(procs)):
        for lvl in range(kw["levels"]):
            assert hc.cell_mismatch(ga.level_of(b, lvl), gw.level_of(b, lvl))[0] == 0, (b, lvl)


def _raw_call(g, n_scans, scans, hints=None, given=False):
    """The C entry point with arbitrary counts (the harness derives them from the lists)."""
    ns = np.asarray(n_scans, np.int32)
    cnt = np.array([len(s) for s in scans], np.int32)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(s, np.float32).reshape(-1, 2) for s in scans]), np.float32)
    out = np.zeros((max(len(scans), 1), 3), np.float32)
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    i = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))  # noqa: E731
    origo = np.zeros(2, np.float32)
    h = np.ascontiguousarray(hints, np.float32) if hints is not None else None
    return g.L.b2s_hector_slam_process_stream_batch(g.h, i(ns), f(cat), i(cnt), f(origo), None,
                                                    f(h) if h is not None else None, int(given), f(out), None, None)


def test_refused_calls_change_nothing(pkg, H):
    """Refused calls leave every processor as it was, and the next valid call still equals the restatement."""
    abi = pkg.abi
    kw = hc.processor_kw("wide")
    walk, bl = hc.make_stream("wide", "walk"), hc.make_stream("wide", "batch_long")
    big = np.concatenate([bl.scans[-1], bl.scans[-1][:1]])  # 4097 points
    assert len(big) == 4097 and len(bl.scans[0]) == 2049
    first, second = _sub(walk, 0, 5), _sub(walk, 5, 10)
    for cap, too_big in ((4096, big), (2048, bl.scans[0])):
        g = H.HectorSlam(batch=2, max_points=cap, **kw)
        g.process_stream_batch([first.scans, first.scans[:2]], (0, 0), pose_hints=[first.hints, first.hints[:2]])
        before = [([g.level_of(b, l) for l in range(3)], g.last_poses(b)) for b in range(2)]
        sc = [walk.scans[6], too_big]
        assert _raw_call(g, [1, 1], sc, np.stack([walk.hints[6]] * 2)) == abi.B2S_ERR_TOO_LARGE, cap
        assert _raw_call(g, [-1, 2], walk.scans[:1], walk.hints[:1]) == abi.B2S_ERR_BAD_PARAMS
        assert _raw_call(g, [1, 1], walk.scans[:2], None, given=True) == abi.B2S_ERR_BAD_PARAMS
        for b in range(2):
            for l in range(3):
                assert hc.cell_mismatch(g.level_of(b, l), before[b][0][l])[0] == 0, (cap, b, l)
            for x, y in zip(g.last_poses(b), before[b][1]):
                assert hc.same_bits(x, y), (cap, b)
        res, covs = g.process_stream_batch([second.scans, second.scans], (0, 0), pose_hints=[second.hints] * 2)
        for b, pre in enumerate((first, _sub(first, 0, 2))):
            c = port.PortHectorProcessor(**kw)
            for i in range(len(pre)):
                c.update(pre.scans[i], (0, 0), pre.hints[i])
            for i in range(len(second)):
                ec, cc = c.update(second.scans[i], (0, 0), second.hints[i])
                assert hc.same_bits(res[b][0][i], ec) and res[b][1][i] == c.map_updated, (cap, b, i)
            assert hc.same_bits(covs[b], cc), (cap, b)
            _levels_equal(g, b, c, 3, ("after refusals", cap, b))
            c.close()
        g.close()


def test_ros_payloads(H):
    """copy_level_ros_of(b) is the ROS rule (log-odds < 0: 0, > 0: 100, else -1) on processor b's plane, on every level;
    copy_level_ros is processor 0's."""
    kw = hc.processor_kw("wide")
    procs = _ragged_fleet()
    g = H.HectorSlam(batch=len(procs), max_points=4096, **kw)
    _fleet_call(g, procs, "self")
    for lvl in range(kw["levels"]):
        for b in range(len(procs)):
            lo = g.level_of(b, lvl)[0]
            want = np.where(lo < 0, 0, np.where(lo > 0, 100, -1)).astype(np.int8)
            assert np.array_equal(g.ros_map_of(b, lvl), want), (b, lvl)
        assert np.array_equal(g.ros_map(lvl), g.ros_map_of(0, lvl)), lvl
    assert (g.ros_map_of(5, 0) == 100).sum() > 100 and (g.ros_map_of(0, 0) == -1).all()
