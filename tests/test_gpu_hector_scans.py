"""GPU tests of b2s_hector_slam_process_scans_batch (k_hs_stream_batch<_, true>): every processor of a handle walks its
own recording of raw LaserScan ranges, each scan converted on the device (projectLaser + rosPointCloudToDataContainer)
inside the fleet launch.

It must equal the host conversion (b2s_ros_hector_scans) followed by b2s_hector_slam_process_stream_batch on a twin
handle: poses, gate flags, last Hessians, last poses, every cell of every level and the kept-beam counts, bit for bit in
exact and fast mode.  One fleet is also checked against the restatement end to end (oracle conversion, then
PortHectorProcessor)."""
import ctypes as C

import numpy as np
import pytest

import hector_cases as hc
from oracle import hector_scans_port as O
from oracle import port

pytestmark = pytest.mark.gpu
f32 = np.float32
LASER = hc.synth.Laser()
LASER_4096 = hc.LONG_LASER
MOUNT = dict(laser_in_base=(0.12, -0.05, 0.2, 0.03))


@pytest.fixture(scope="module")
def H(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector")


@pytest.fixture(scope="module")
def R(pkg):
    return pkg.load("rosio")


def _geometry(R, laser):
    amin, inc = f32(laser.min_angle), f32(laser.angular_resolution)
    return R.make_msg(amin, amin + inc * f32(laser.n_readings - 1), inc, 0.1, 30.0, np.zeros(laser.n_readings, np.float32))


def _recording(seed, n, laser=LASER, dropout=0.0):
    """n scans of a walk: float32 ranges [n, beams] and the true poses (the hints)."""
    _, poses, ranges = hc.synth.make_trajectory(seed, n, laser, step_xy=0.1, step_th_deg=3)
    r = ranges.astype(np.float32)
    if dropout:
        rng = np.random.default_rng(seed)
        bad = rng.random(r.shape) < dropout
        r[bad] = rng.choice(np.array([np.nan, np.inf, -np.inf, 0.0, 0.05], np.float32), int(bad.sum()))
    return r, poses.astype(np.float32)


def _ragged(laser=LASER):
    """(ranges, hints) per processor: no scans, one scan, only dropouts, dropout-heavy, two plain walks."""
    walk_r, walk_h = _recording(7, 8, laser)
    empty = np.full((3, laser.n_readings), np.nan, np.float32)
    heavy_r, heavy_h = _recording(8, 6, laser, dropout=0.6)
    other_r, other_h = _recording(9, 7, laser)
    return [(walk_r[:0], walk_h[:0]), (walk_r[:1], walk_h[:1]), (empty, walk_h[:3]), (heavy_r, heavy_h),
            (walk_r, walk_h), (other_r, other_h)]


def _hint_args(procs, form, first_hints=True):
    firsts = np.stack([h[0] if len(h) else np.zeros(3, np.float32) for _, h in procs])
    if form == "self":
        return dict(first_hints=firsts if first_hints else None)
    return dict(pose_hints=[h for _, h in procs], map_without_matching=form == "given")


def _host_points(R, geom, procs, filt, scale):
    streams, kept, origo = [], [], None
    for r, _ in procs:
        pts, cnt, origo = R.hector_scans(geom, r, filt, scale)
        edges = np.concatenate([[0], np.cumsum(cnt)])
        streams.append([pts[edges[i]:edges[i + 1]] for i in range(len(cnt))])
        kept.append(cnt)
    return streams, kept, origo


def _assert_twins(ga, gb, ra, rb, ca, cb, levels, what):
    for b in range(len(ra)):
        assert hc.same_bits(ra[b][0], rb[b][0]) and np.array_equal(ra[b][1], rb[b][1]), (what, b)
        for x, y in zip(ga.last_poses(b), gb.last_poses(b)):
            assert hc.same_bits(x, y), (what, b)
        for lvl in range(levels):
            assert hc.cell_mismatch(ga.level_of(b, lvl), gb.level_of(b, lvl))[0] == 0, (what, b, lvl)
    assert hc.same_bits(ca, cb), what


def _device_vs_host(H, R, procs, laser, form, exact, cap, filt_kw=MOUNT, geometry="wide"):
    kw = hc.processor_kw(geometry)
    geom, filt = _geometry(R, laser), R.hector_scan_filter(**filt_kw)
    scale = f32(1.0) / f32(kw["resolution"])
    B = len(procs)
    ga = H.HectorSlam(batch=B, max_points=cap, exact=exact, **kw)
    gb = H.HectorSlam(batch=B, max_points=cap, exact=exact, **kw)
    ra, ca, kept = ga.process_scans_batch(geom, [r for r, _ in procs], filt, **_hint_args(procs, form))
    streams, want_kept, origo = _host_points(R, geom, procs, filt, scale)
    rb, cb = gb.process_stream_batch(streams, origo, **_hint_args(procs, form))
    what = (form, exact, cap, B)
    for b in range(B):
        assert np.array_equal(kept[b], want_kept[b]), (what, b)
    _assert_twins(ga, gb, ra, rb, ca, cb, kw["levels"], what)
    ga.close(), gb.close()
    return kept


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("form", ["self", "hints", "given"])
def test_ragged_fleet_equals_host_conversion(H, R, form, exact):
    kept = _device_vs_host(H, R, _ragged(), LASER, form, exact, 2048)
    assert len(kept[0]) == 0 and len(kept[1]) == 1 and not kept[2].any() and kept[3].all() and kept[4].all()


@pytest.mark.parametrize("exact", [True, False])
def test_4096_beams_at_capacity(H, R, exact):
    """n_ranges = max_points = 4096: one ingest round of 576 beams is not enough seven times over."""
    procs = [_recording(11, 4, LASER_4096), _recording(12, 3, LASER_4096, dropout=0.3)]
    for form in ("self", "given"):
        kept = _device_vs_host(H, R, procs, LASER_4096, form, exact, 4096, filt_kw=dict(laser_in_base=(0.0, 0.0, 0.0, 0.0)))
        assert kept[0].max() > 2048


@pytest.mark.parametrize("exact", [True, False])
def test_single_processor(H, R, exact):
    _device_vs_host(H, R, [_recording(13, 5)], LASER, "self", exact, 2048)


def test_300_processors(H, R):
    base = [_recording(20 + k, 4) for k in range(5)]
    procs = []
    for b in range(300):
        r, h = base[b % 5]
        lo, n = b % 3, (b // 5) % 3  # 0, 1 or 2 scans from one of three starting points
        procs.append((r[lo:lo + n], h[lo:lo + n]))
    _device_vs_host(H, R, procs, LASER, "self", True, 2048)
    _device_vs_host(H, R, procs, LASER, "hints", False, 2048)


@pytest.mark.parametrize("exact", [True, False])
def test_split_calls_equal_one(H, R, exact):
    kw = hc.processor_kw("wide")
    geom, filt = _geometry(R, LASER), R.hector_scan_filter(**MOUNT)
    procs = _ragged()
    cut = [0, 0, 2, 3, 5, 1]
    ga = H.HectorSlam(batch=len(procs), max_points=2048, exact=exact, **kw)
    gb = H.HectorSlam(batch=len(procs), max_points=2048, exact=exact, **kw)
    ra1, _, _ = ga.process_scans_batch(geom, [r[:c] for (r, _), c in zip(procs, cut)], filt, **_hint_args(procs, "self"))
    # the second part chains through each processor's last scan-match pose, except where the first part was empty
    rest = [(r[c:], h[c:]) for (r, h), c in zip(procs, cut)]
    first = np.stack([ra1[b][0][-1] if cut[b] else (rest[b][1][0] if len(rest[b][1]) else np.zeros(3, np.float32))
                      for b in range(len(procs))])
    ra2, ca, _ = ga.process_scans_batch(geom, [r for r, _ in rest], filt, first_hints=first)
    rb, cb, _ = gb.process_scans_batch(geom, [r for r, _ in procs], filt, **_hint_args(procs, "self"))
    for b in range(len(procs)):
        assert hc.same_bits(np.concatenate([ra1[b][0], ra2[b][0]]), rb[b][0]), b
        assert np.array_equal(np.concatenate([ra1[b][1], ra2[b][1]]), rb[b][1]), b
        for x, y in zip(ga.last_poses(b), gb.last_poses(b)):
            assert hc.same_bits(x, y), b
        for lvl in range(kw["levels"]):
            assert hc.cell_mismatch(ga.level_of(b, lvl), gb.level_of(b, lvl))[0] == 0, (b, lvl)
        if len(rest[b][0]):
            assert hc.same_bits(ca[b], cb[b]), b
    ga.close(), gb.close()


def test_fleet_against_the_restatement(H, R):
    """Oracle conversion of every scan, then PortHectorProcessor over each processor's scans."""
    kw = hc.processor_kw("wide")
    geom = _geometry(R, LASER)
    filt_kw = dict(laser_in_base=(0.1, 0.05, 0.3, -0.04), min_dist=0.25, max_dist=25.0, use_max_scan_range=15.0)
    procs = [_recording(31, 4), _recording(32, 3, dropout=0.4), (np.zeros((0, LASER.n_readings), f32), np.zeros((0, 3), f32))]
    g = H.HectorSlam(batch=3, max_points=2048, **kw)
    res, covs, kept = g.process_scans_batch(geom, [r for r, _ in procs], R.hector_scan_filter(**filt_kw),
                                            **_hint_args(procs, "self"))
    scale = f32(1.0) / f32(kw["resolution"])
    for b, (r, h) in enumerate(procs):
        dcs, origo = O.scans(r, geom.angle_min, geom.angle_increment, geom.range_min, geom.range_max, 30.0, scale, **filt_kw)
        assert list(kept[b]) == [len(d) for d in dcs], b
        c = port.PortHectorProcessor(**kw)
        est, cc = (h[0] if len(h) else None), None
        for i, pts in enumerate(dcs):
            est, cc = c.update(pts, origo, est)
            assert hc.same_bits(res[b][0][i], est) and res[b][1][i] == c.map_updated, (b, i)
        if len(dcs):
            assert hc.same_bits(covs[b], cc), b
        else:
            assert not covs[b].any()
        for lvl in range(kw["levels"]):
            assert hc.cell_mismatch(g.level_of(b, lvl), c.level(lvl))[0] == 0, (b, lvl)
        c.close()
    g.close()


def _raw(g, geom, filt, n_scans, ranges, given=False, hints=None):
    ns = np.asarray(n_scans, np.int32)
    r = np.ascontiguousarray(ranges, np.float32) if ranges is not None else None
    total = max(int(np.clip(ns, 0, None).sum()), 1)
    out = np.zeros((total, 3), np.float32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    h = np.ascontiguousarray(hints, np.float32) if hints is not None else None
    return g.L.b2s_hector_slam_process_scans_batch(g.h, C.byref(geom) if geom is not None else None,
                                                   C.byref(filt) if filt is not None else None, ns.ctypes.data_as(ip),
                                                   r.ctypes.data_as(fp) if r is not None else None, None,
                                                   h.ctypes.data_as(fp) if h is not None else None, int(given),
                                                   out.ctypes.data_as(fp), None, None, None)


def test_refused_calls_change_nothing(pkg, H, R):
    abi = pkg.abi
    kw = hc.processor_kw("wide")
    geom, filt = _geometry(R, LASER), R.hector_scan_filter(**MOUNT)
    r, h = _recording(41, 6)
    g = H.HectorSlam(batch=2, max_points=2048, **kw)
    g.process_scans_batch(geom, [r[:3], r[:2]], filt, first_hints=np.stack([h[0], h[0]]))  # binds the argument types
    before = [([g.level_of(b, l) for l in range(3)], g.last_poses(b)) for b in range(2)]
    long_geom, long_r = _geometry(R, LASER_4096), _recording(42, 2, LASER_4096)[0]
    assert _raw(g, long_geom, filt, [1, 1], long_r) == abi.B2S_ERR_TOO_LARGE
    assert _raw(g, geom, filt, [-1, 2], r[:1]) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(g, geom, filt, [1, 1], None) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(g, None, filt, [1, 1], r[:2]) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(g, geom, None, [1, 1], r[:2]) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(g, geom, filt, [1, 1], r[:2], given=True) == abi.B2S_ERR_BAD_PARAMS
    for b in range(2):
        for lvl in range(3):
            assert hc.cell_mismatch(g.level_of(b, lvl), before[b][0][lvl])[0] == 0, (b, lvl)
        for x, y in zip(g.last_poses(b), before[b][1]):
            assert hc.same_bits(x, y), b
    # and the next valid call continues both processors as if nothing had been refused
    g2 = H.HectorSlam(batch=2, max_points=2048, **kw)
    g2.process_scans_batch(geom, [r[:3], r[:2]], filt, first_hints=np.stack([h[0], h[0]]))
    ra, ca, _ = g.process_scans_batch(geom, [r[3:], r[2:]], filt)
    rb, cb, _ = g2.process_scans_batch(geom, [r[3:], r[2:]], filt)
    _assert_twins(g, g2, ra, rb, ca, cb, 3, "after refusals")
    g.close(), g2.close()
