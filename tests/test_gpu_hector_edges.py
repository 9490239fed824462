"""GPU tests of the Hector processor (hector_slam.cu) and the single-map handle (hector_map.cu) on the edge cases of
tests/hector_cases.py: non-square maps both ways, a robot near two edges of the map, 1, 4 and 8 levels, a 12 x 12 map,
scans of 0 ... 4096 points, crafted stamp-order rays and match points on the interpolation limit.

The restatement (PortHectorProcessor) is the reference here; it is pinned to the unmodified lesson4 headers on the same
cases by tests/test_hector_edges_reference.py, and where that build travelled with the repository (oracle/_ref) the
device is compared with it directly as well.  Exact mode: poses, Hessians, gate decisions and every cell of every level
bit for bit (a NaN pose matches a NaN pose; x86 and the GPU write different NaN payloads)."""
import numpy as np
import pytest

import hector_cases as hc
from oracle import port

pytestmark = pytest.mark.gpu
DEVICE_FAMILIES = [f for f in hc.FAMILIES if f != "batch_long"]  # the single handle holds 2048 points


@pytest.fixture(scope="module")
def H(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector")


def _cpu_processors(kw, reference_ok):
    from oracle import ref_hector as rh
    out = [("restatement", port.PortHectorProcessor(**kw))]
    if reference_ok and rh.available():
        out.append(("reference", rh.RefHectorProcessor(**kw)))
    return out


def _device_stream(g, stream, form):
    if form == "self":
        return g.process_stream(stream.scans, (0, 0), first_hint=stream.first)
    return g.process_stream(stream.scans, (0, 0), pose_hints=stream.hints, map_without_matching=form == "given")


def _levels_equal(g, c, levels, what, b=None):
    for lvl in range(levels):
        bad, touched = hc.cell_mismatch(g.level(lvl) if b is None else g.level_of(b, lvl), c.level(lvl))
        assert bad == 0, (what, lvl, bad, touched)


@pytest.mark.parametrize("family", DEVICE_FAMILIES)
@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_exact_streams(H, geometry, family):
    """update() per scan and process_stream, each in the three forms, against the CPU processor and each other."""
    kw = hc.processor_kw(geometry)
    stream = hc.make_stream(geometry, family)
    for form in hc.FORMS[family]:
        cpus = _cpu_processors(kw, reference_ok=True)
        ref = {}
        for name, c in cpus:
            if name == "reference" and np.isnan(ref["restatement"][0]).any():
                break  # the reference's interpolation at a NaN coordinate is undefined (test_hector_edges_reference)
            ref[name] = hc.run_stream(c, stream, form)
        pc, cc, fc = ref["restatement"]
        g = H.HectorSlam(**kw)
        pg, cg, fg = hc.run_stream(g, stream, form)
        assert hc.same_bits(pg, pc), (form, np.flatnonzero(~((pg == pc) | (np.isnan(pg) & np.isnan(pc))).all(1)))
        assert hc.same_bits(cg, cc), form
        assert np.array_equal(fg, fc), (form, fg, fc)
        if "reference" in ref:
            assert hc.same_bits(pg, ref["reference"][0]) and hc.same_bits(cg, ref["reference"][1]), form
        g2 = H.HectorSlam(**kw)
        ps, us, cov_last = _device_stream(g2, stream, form)
        assert hc.same_bits(ps, pc) and np.array_equal(us, fc), form
        if form != "given":
            assert hc.same_bits(cov_last, cc[-1]), form
        a, _ = g2.last_poses()
        assert hc.same_bits(a, pc[-1])
        for name, c in cpus:
            if name in ref:
                _levels_equal(g, c, kw["levels"], (form, name, "update"))
                _levels_equal(g2, c, kw["levels"], (form, name, "process_stream"))
            c.close()
        g.close(), g2.close()


def test_single_handle_capacity(pkg, H):
    """2048 points are accepted (the long family ends on them); 2049 are refused with B2S_ERR_TOO_LARGE and change
    nothing, and the next valid call still equals the CPU processor."""
    M = pkg.load("matcher")
    kw = hc.processor_kw("wide")
    s = hc.make_stream("wide", "long")
    big = hc.make_stream("wide", "batch_long").scans[0]
    assert len(big) == 2049 and len(s.scans[-1]) == 2048
    g, c = H.HectorSlam(**kw), port.PortHectorProcessor(**kw)
    for i in range(len(s) - 2, len(s)):
        eg, _ = g.update(s.scans[i], (0, 0), s.hints[i])
        ec, _ = c.update(s.scans[i], (0, 0), s.hints[i])
        assert hc.same_bits(eg, ec)
    before = [g.level(l) for l in range(3)], g.last_poses()
    with pytest.raises(M.B2SError) as e:
        g.update(big, (0, 0), s.hints[0])
    assert e.value.status == pkg.abi.B2S_ERR_TOO_LARGE
    with pytest.raises(M.B2SError) as e:
        g.process_stream([s.scans[0], big], (0, 0), first_hint=s.first)
    assert e.value.status == pkg.abi.B2S_ERR_TOO_LARGE
    for l in range(3):
        assert hc.cell_mismatch(g.level(l), before[0][l])[0] == 0
    after = g.last_poses()
    assert hc.same_bits(after[0], before[1][0]) and hc.same_bits(after[1], before[1][1])
    eg, cg = g.update(s.scans[-1], (0, 0), s.hints[3])
    ec, cc = c.update(s.scans[-1], (0, 0), s.hints[3])
    assert hc.same_bits(eg, ec) and hc.same_bits(cg, cc) and g.map_updated == c.map_updated
    _levels_equal(g, c, 3, "after the refused call")


def test_create_limits(pkg, H):
    M = pkg.load("matcher")
    with pytest.raises(M.B2SError) as e:
        H.HectorSlam(batch=2, max_points=4097, **hc.GEOMETRIES["wide"])
    assert e.value.status == pkg.abi.B2S_ERR_TOO_LARGE
    H.HectorSlam(batch=1, max_points=4096, **hc.GEOMETRIES["wide"]).close()
    for sx, sy in ((11, 12), (12, 11)):  # 11 >> 2 = 2: the first size below the 3-level floor
        with pytest.raises(M.B2SError) as e:
            H.HectorSlam(**dict(hc.GEOMETRIES["tiny"], size_x=sx, size_y=sy))
        assert e.value.status == pkg.abi.B2S_ERR_BAD_PARAMS
    with pytest.raises(M.B2SError):
        H.HectorSlam(**dict(hc.GEOMETRIES["deep"], levels=9))
    g = H.HectorSlam(**hc.GEOMETRIES["tiny"])
    assert [g.level_dims(l)[:2] for l in range(3)] == [(12, 12), (6, 6), (3, 3)]


def _ragged_batch():
    """Five processors on the wide map, four steps: 0 points, 1 ... 4 points, 2049 ... 4096 points, the wide walk and
    the edge map's walk (same resolution)."""
    walk = hc.make_stream("wide", "walk")
    edge = hc.make_stream("edge", "walk")
    longs = hc.make_stream("wide", "long")
    bl = hc.make_stream("wide", "batch_long")
    steps = 4
    scans = [[np.zeros((0, 2), np.float32)] * steps, longs.scans[:steps], bl.scans, walk.scans[:steps], edge.scans[:steps]]
    hints = np.stack([walk.hints[:steps] * np.float32(0.5), longs.hints[:steps], bl.hints, walk.hints[:steps],
                      edge.hints[:steps]], 1)  # [step][b][3]
    return scans, hints


def _cpu_batch(kw, scans, hints, chain=False):
    """Each processor of the batch on its own CPU processor: hints given, or (chain) the first step's hint and then the
    last scan-match pose."""
    out = []
    for b in range(len(scans)):
        c = port.PortHectorProcessor(**kw)
        est, poses, covs, flags = hints[0, b], [], [], []
        for i in range(len(scans[b])):
            est, cov = c.update(scans[b][i], (0, 0), est if chain else hints[i, b])
            poses.append(est), covs.append(cov), flags.append(c.map_updated)
        out.append((c, np.stack(poses), np.stack(covs), np.array(flags)))
    return out


def test_batch_ragged_equals_single_and_restatement(pkg, H):
    kw = hc.processor_kw("wide")
    scans, hints = _ragged_batch()
    B, steps = len(scans), len(scans[0])
    gb = H.HectorSlam(batch=B, max_points=4096, **kw)
    singles = {b: H.HectorSlam(**kw) for b in (0, 1, 3, 4)}  # (processor 2's scans exceed the single handle)
    cpu = _cpu_batch(kw, scans, hints)
    for i in range(steps):
        pb, cb, ub = gb.update_batch([scans[b][i] for b in range(B)], (0, 0), hints[i])
        for b in range(B):
            _, pc, cc, fc = cpu[b]
            assert hc.same_bits(pb[b], pc[i]) and ub[b] == fc[i], (i, b, pb[b], pc[i])
            if len(scans[b][i]):
                assert hc.same_bits(cb[b], cc[i]), (i, b)
            if b in singles:
                e1, c1 = singles[b].update(scans[b][i], (0, 0), hints[i, b])
                assert hc.same_bits(pb[b], e1) and ub[b] == singles[b].map_updated, (i, b)
    for b in range(B):
        _levels_equal(gb, cpu[b][0], 3, ("restatement", b), b=b)
        if b in singles:
            _levels_equal(gb, singles[b], 3, ("single", b), b=b)
    assert (gb.level_of(2, 0)[1] >= 0).sum() > 1000 and (gb.level_of(0, 0)[1] >= 0).sum() == 0


@pytest.mark.parametrize("with_hints", [True, False])
def test_batch_device_pointers_equal_host_batch(pkg, H, with_hints):
    """update_batch_device with the points, counts and hints in torch CUDA tensors (or no hints: the chain through the
    last match pose) leaves last_poses and every level equal to the update_batch twin's; the chained run also equals
    the CPU processors."""
    import torch
    kw = hc.processor_kw("wide")
    scans, hints = _ragged_batch()
    B, steps, cap = len(scans), len(scans[0]), 4096
    gh, gd = H.HectorSlam(batch=B, max_points=cap, **kw), H.HectorSlam(batch=B, max_points=cap, **kw)
    if not with_hints:  # both chains start from the same pose: one step with hints, then none
        gh.update_batch([scans[b][0] for b in range(B)], (0, 0), hints[0])
        gd.update_batch([scans[b][0] for b in range(B)], (0, 0), hints[0])
    for i in range(0 if with_hints else 1, steps):
        step = [scans[b][i] for b in range(B)]
        gh.update_batch(step, (0, 0), hints[i] if with_hints else None)
        pts = np.zeros((B, cap, 2), np.float32)
        for b, s in enumerate(step):
            pts[b, :len(s)] = s
        cnt = np.array([len(s) for s in step], np.int32)
        d_pts, d_cnt = torch.from_numpy(pts).cuda(), torch.from_numpy(cnt).cuda()
        d_h = torch.from_numpy(np.ascontiguousarray(hints[i])).cuda() if with_hints else None
        torch.cuda.synchronize()
        gd.update_batch_device(d_pts.data_ptr(), d_cnt.data_ptr(), int(cnt.max()), (0, 0),
                               d_h.data_ptr() if with_hints else None)
        gd.sync()
    for b in range(B):
        for x, y in zip(gd.last_poses(b), gh.last_poses(b)):
            assert hc.same_bits(x, y), b
        for lvl in range(3):
            assert hc.cell_mismatch(gd.level_of(b, lvl), gh.level_of(b, lvl))[0] == 0, (b, lvl)
    if not with_hints:
        cpu = _cpu_batch(kw, scans, hints, chain=True)
        for b in range(B):
            assert hc.same_bits(gh.last_poses(b)[0], cpu[b][1][-1]), b
            _levels_equal(gh, cpu[b][0], 3, ("chain", b), b=b)


def test_batch_epoch_wrap(pkg, H):
    """Crossing the 20-bit stamp epoch on the batched handle changes nothing."""
    kw = hc.processor_kw("wide")
    scans, hints = _ragged_batch()
    B, steps = len(scans), len(scans[0])
    ga, gw = H.HectorSlam(batch=B, max_points=4096, **kw), H.HectorSlam(batch=B, max_points=4096, **kw)
    for i in range(steps):
        if i == 1:
            gw.debug_set_epoch((1 << 20) - 3)
        step = [scans[b][i] for b in range(B)]
        pa, ca, ua = ga.update_batch(step, (0, 0), hints[i], map_without_matching=i % 2 == 0)
        pw, cw, uw = gw.update_batch(step, (0, 0), hints[i], map_without_matching=i % 2 == 0)
        assert hc.same_bits(pa, pw) and hc.same_bits(ca, cw) and np.array_equal(ua, uw), i
    for b in range(B):
        for lvl in range(3):
            assert hc.cell_mismatch(ga.level_of(b, lvl), gw.level_of(b, lvl))[0] == 0, (b, lvl)


def _fast_scans():
    s = hc.make_stream("wide", "long")
    w = hc.make_stream("wide", "walk")
    return s.scans + w.scans, np.concatenate([s.hints, w.hints])


def test_fast_batch_equals_one_cta_stream(pkg, H, monkeypatch):
    """Fast mode, batched (k_hs_match<false>) and single with B2S_HS_CLUSTER=0 (k_hs_stream<false, false>): both run
    hs_match_cta<false, false> on the same scans and hints, so they agree bit for bit."""
    kw = dict(hc.processor_kw("wide"), min_dist=1e9, min_angle=1e9)  # one map for every scan: the gate stays shut
    scans, hints = _fast_scans()
    monkeypatch.setenv("B2S_HS_CLUSTER", "0")
    g1 = H.HectorSlam(exact=False, **kw)
    monkeypatch.delenv("B2S_HS_CLUSTER")
    assert g1.cluster_size() == 1
    gb = H.HectorSlam(exact=False, batch=1, max_points=2048, **kw)
    c = port.PortHectorProcessor(**kw)
    w = hc.make_stream("wide", "walk")
    for g in (g1, c):
        for i in range(4):
            g.update(w.scans[i], (0, 0), w.hints[i], True)
    gb.update_batch(w.scans[:1], (0, 0), w.hints[:1], True)
    for i in range(1, 4):
        gb.update_batch(w.scans[i:i + 1], (0, 0), w.hints[i:i + 1], True)
    for i in range(len(scans)):
        e1, c1 = g1.update(scans[i], (0, 0), hints[i])
        pb, cb, ub = gb.update_batch([scans[i]], (0, 0), hints[i][None])
        assert hc.same_bits(pb[0], e1) and hc.same_bits(cb[0], c1) and ub[0] == g1.map_updated, (i, len(scans[i]))
        ec, _ = c.update(scans[i], (0, 0), hints[i])
        if len(scans[i]) >= 575:  # (a few points give a near-singular Hessian: there the tree sum may take another path)
            assert np.abs(e1 - ec).max() <= 1e-4, (i, e1, ec)
    for lvl in range(3):
        assert hc.cell_mismatch(gb.level_of(0, lvl), g1.level(lvl))[0] == 0, lvl


def test_fast_cluster_uneven_shares(pkg, H, monkeypatch):
    """The clustered fast stream splits a scan over 4 CTAs (hs_share): empty and uneven shares for n = 1 ... 9, 33,
    1153, 2048.  Poses within the 1e-4 contract of the restatement; gate decisions equal the one-CTA path's."""
    # the gate stays shut after the mapping-only warm-up, so every cut scan is matched against the same map
    kw = dict(hc.processor_kw("wide"), min_dist=1e9, min_angle=1e9)
    gc = H.HectorSlam(exact=False, **kw)
    if gc.cluster_size() != 4:
        pytest.skip("thread-block cluster launch not available here: the fast path runs on one CTA")
    monkeypatch.setenv("B2S_HS_CLUSTER", "0")
    g1 = H.HectorSlam(exact=False, **kw)
    monkeypatch.delenv("B2S_HS_CLUSTER")
    s = hc.make_stream("wide", "long")
    lengths = (1, 2, 3, 4, 5, 6, 7, 8, 9, 33, 1153, 2048)
    src = s.scans[-1]  # 2048 points
    # map the room from the last poses first (mapping only), then match the cut scans from the last pose
    for g in (gc, g1):
        g.process_stream(s.scans[-4:], (0, 0), pose_hints=s.hints[-4:], map_without_matching=True)
    c = port.PortHectorProcessor(**kw)
    for i in range(len(s) - 4, len(s)):
        c.update(s.scans[i], (0, 0), s.hints[i], True)
    scans = [np.ascontiguousarray(src[:n]) for n in lengths]
    ph = np.repeat(s.hints[-1:], len(scans), 0)
    pc_, uc, _ = gc.process_stream(scans, (0, 0), pose_hints=ph)
    p1, u1, _ = g1.process_stream(scans, (0, 0), pose_hints=ph)
    ref = np.stack([c.update(sc, (0, 0), ph[i])[0] for i, sc in enumerate(scans)])
    ok = ~np.isnan(ref).any(1)
    assert np.array_equal(np.isnan(pc_).any(1), ~ok)
    assert np.abs(pc_[ok] - ref[ok]).max() <= 1e-4 and np.abs(pc_[ok] - p1[ok]).max() <= 1e-4
    assert list(uc) == list(u1)


@pytest.mark.parametrize("geometry", ["wide", "tall_odd", "edge"])
def test_single_map_handle_non_square(pkg, H, geometry):
    """HectorMap (hector_map.cu) on the non-square and edge geometries: update cells bit for bit, match_data within
    its documented 1e-4."""
    gm = hc.GEOMETRIES[geometry]
    sx, sy, res, (stx, sty) = gm["size_x"], gm["size_y"], gm["resolution"], gm["start"]
    s = hc.make_stream(geometry, "walk")
    g, c = H.HectorMap(sx, sy, res, stx, sty), port.PortHectorMap(sx, sy, res, stx, sty)
    g.set_factors(0.4, 0.9), c.set_factors(0.4, 0.9)
    for i in range(len(s) - 1):
        g.update_by_scan(s.scans[i], (0, 0), s.hints[i])
        c.update_by_scan(s.scans[i], (0, 0), s.hints[i])
    assert hc.cell_mismatch(g.cells(), c.cells())[0] == 0
    st = hc.make_stream(geometry, "stamps")
    for i in range(len(st)):
        g.update_by_scan(st.scans[i], (0, 0), st.hints[i])
        c.update_by_scan(st.scans[i], (0, 0), st.hints[i])
    bad, touched = hc.cell_mismatch(g.cells(), c.cells())
    assert bad == 0 and touched > 1000
    start = (s.hints[-1] + np.array([0.03, -0.02, 0.01], np.float32)).astype(np.float32)
    eg, _ = g.match_data(s.scans[-1], start, 5)
    ec, _ = c.match_data(s.scans[-1], start, 5)
    assert np.abs(eg - ec).max() <= 1e-4, (eg, ec)
    ie = hc.make_stream(geometry, "interp_edge")
    eg, _ = g.match_data(ie.scans[0], ie.hints[0], 3)
    ec, _ = c.match_data(ie.scans[0], ie.hints[0], 3)
    assert np.abs(eg - ec).max() <= 1e-4 or (np.isnan(eg).all() and np.isnan(ec).all()), (eg, ec)


def test_batch_stamps_past_2048(pkg, H):
    """Beams 2048 ... 4095 keep their own stamps (12-bit beam field): beam 0 ends on a cell that beam 2048 crosses
    (no un-free), beam 1 crosses a cell that beam 2049 ends on (un-free).  Zero-length rays fill the indices between;
    the scan is applied four times with update factors 0.35 / 0.8, where the "(v + f) - f" rounding shows in the
    log-odds from the third."""
    kw = dict(hc.processor_kw("wide"), update_free=0.35, update_occupied=0.8)
    r = (100, 100)
    a1, b1, a2, b2 = (104, 100), (106, 100), (100, 104), (100, 106)
    ends = [a1, b2] + [r] * 2046 + [b1, a2]
    w = hc._world_of("wide", *r)
    mx, my = hc._map_of("wide", w)
    pts = np.array([(e[0] - float(mx), e[1] - float(my)) for e in ends], np.float32)
    assert len(pts) == 2050
    g = H.HectorSlam(batch=2, max_points=4096, **kw)
    c = port.PortHectorProcessor(**kw)
    for _ in range(4):
        g.update_batch([pts, pts[:2]], (0, 0), np.stack([w, w]), map_without_matching=True)
        c.update(pts, (0, 0), w, True)
    _levels_equal(g, c, 3, "stamps past 2048", b=0)
    lo, ui = c.level(0)
    assert ui[a1[1], a1[0]] == ui[a2[1], a2[0]] and lo[a1[1], a1[0]] != lo[a2[1], a2[0]]  # the un-free rounding shows
