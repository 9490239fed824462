"""The bounds behind the correlative sweep's angle pruning, read back per match (b2s_matcher_last_prune_state) and
checked against the dense volume and the numpy restatements, on the device.

For every match the pruned path took:
  1. soundness: the largest exact response of each angle k is <= gub[k // 4], and <= ubr[k] where ubr[k] is set;
  2. ubr[k], where the device set it, equals the numpy single-angle bound (tests/test_prune_bound.py) bit for bit;
  3. gub[g] >= the numpy bound of every member, evaluated or not, and equals the fp32 group-bracket restatement
     (tests/group_bracket_reference.py) except in groups it flags borderline;
  4. the numpy rounds (tests/test_prune_group_bound.py) on the numpy ubr and the device's gub give exactly the angles
     the device bounded one by one and the angles it swept, and cut = L - 0.1 - 1e-9 with L the best exact response
     of the probe;
  5. every angle left out has all its exact responses below cut, and last_pruned_frac() is the unswept share;
  6. pruned results equal dense ones byte for byte.
The responses come from the device's own integer volume (response_sums), which the other tests hold equal to the
restatement's.  A match the generic kernel takes reads back ubr and cut NaN and every angle swept.

The cases: the benchmark's shape at 1024 matches with and without the penalty (2 - 4 on a seeded sample of 64); rounds
(c) of 17 - 31, exactly 31, exactly 32 and more than 64 angles; beams at the fp32 brackets' edges (spreads of 3 and 4
cells, members near a .5 tie, the 8192-cell cut-off, NaN / inf readings, low corners in the range-tested band and
wholly outside on both sides, grid offsets of 1e5 m); grids of uniform 4 x 4 and 7 x 7 blocks; and an irregular lattice among pruned matches."""
import math

import numpy as np
import pytest

import group_bracket_reference as gr
import karto_volume_reference as kv
from karto_volume_reference import D, abi, port, synth
from test_prune_bound import INVALID, angle_bounds, responses, walls
from test_prune_group_bound import GROUP, rounds

pytestmark = pytest.mark.gpu
SAMPLE = 64


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


# ---------------------------------------------------------------- what a match is checked against


class Ctx:
    """the restatement's inputs of one match: grid, lookup table, first candidate, scan-local points, grid offset"""

    def __init__(self, grid, g, lut, base00, pts, sp, off, ch):
        self.grid, self.g, self.lut, self.base00, self.ch = grid, g, lut, base00, ch
        self.lx, self.ly = gr.local_points(pts, sp)
        self.gox, self.goy = off


def batch_ctx(bt, se):
    def ctx(b):
        gx, gy = bt.cells(b, se)
        if not kv.is_regular(gx, gy, 1):
            return None
        pm = bt._pm(b)
        return Ctx(bt.grids[b], bt.g, bt.lut(b, se), int(gx[0, 0] + gy[0, 0] * bt.g.width_step), pm.pts, pm.sp,
                   bt.offs[b], bt.centers[b][2])
    return ctx


def dropped(c, nx, ny):
    from test_gpu_matcher_prune_lists import dropped_beams
    return dropped_beams(c.grid, c.g, c.lut, c.base00, nx, ny)[0]


def deep_check(c, st_b, resp, n, se, params):
    """invariants 2 - 4 of one match; -> dict(round_c: the angles of round (c) the device bounded, ubr: the numpy
    bound of every angle)"""
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    ubr_d, gub_d, swept, cut = st_b
    na = len(ubr_d)
    ubr = angle_bounds(c.grid, c.g.width_step, np.where(dropped(c, nx, ny), INVALID, c.lut), c.base00, n, se, params,
                       c.ch)
    set_ = ~np.isnan(ubr_d)
    assert np.array_equal(ubr_d[set_].view(np.int64), ubr[set_].view(np.int64)), np.flatnonzero(ubr_d[set_] != ubr[set_])
    assert (gub_d[np.arange(na) // GROUP] >= ubr).all()
    scale = 1.0 / params.resolution
    br = gr.Brackets(c.lx, c.ly, c.ch, se.angle_offset, se.angle_res, na, c.gox, c.goy, scale)
    gub = gr.group_bounds(c.grid, c.g, c.lut, c.base00, n, se, params, c.ch, br)
    border = br.borderline.any(axis=1)
    assert np.array_equal(gub_d[~border], gub[~border]), np.flatnonzero((gub_d != gub) & ~border)
    probe, keep, evs = rounds(ubr, gub_d, resp)
    assert set(np.flatnonzero(set_)) == evs
    assert np.array_equal(swept, keep)
    assert cut == resp[:, :, probe].max() - 0.1 - 1e-9
    _, _, ev_ab = rounds(ubr, gub_d, np.zeros_like(resp))  # rounds (a) and (b) alone: L = 0 keeps every angle
    return dict(round_c=sorted(evs - ev_ab), ubr=ubr)


def check_pruned(m, centers, se, n, params, ctx=None, sample=()):
    """a pruned call, its read-back, the dense volume, invariants 1 and 5 on every match and 2 - 4 on `sample`, then
    pruned == dense (6).  Every match on the pruned path is a regular lattice, so each sampled one is deep-checked.
    -> ({match: deep_check's dict} of the sample, pruned fraction, state)"""
    from test_gpu_matcher_prune import pruned_and_dense
    _, frac_pd = pruned_and_dense(m, centers, se)
    m.correlate_scan(centers, se)
    st = m.last_prune_state()
    frac = m.last_pruned_frac()
    assert frac == frac_pd
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    na = abi.n_steps(se.angle_offset, se.angle_res)
    B = len(centers)
    unswept, sizes = 0, {}
    for b in range(B):
        ubr_d, gub_d, swept, cut = st["ubr"][b], st["gub"][b], st["swept"][b], st["cut"][b]
        if math.isnan(cut):  # the generic kernel
            assert swept.all() and np.isnan(ubr_d).all()
            continue
        resp = responses(m.response_sums(b, (ny, nx, na)), n, se, params, centers[b][2])
        best = resp.reshape(-1, na).max(axis=0)
        assert (best <= gub_d[np.arange(na) // GROUP]).all(), b
        set_ = ~np.isnan(ubr_d)
        assert (best[set_] <= ubr_d[set_]).all(), b
        assert (best[~swept] < cut).all(), b
        unswept += int((~swept).sum())
        if b in sample:
            c = ctx(b)
            assert c is not None, b
            sizes[b] = deep_check(c, (ubr_d, gub_d, swept, cut), resp, n, se, params)
            sizes[b]["best"] = best
    assert frac == unswept / (float(B) * na), (frac, unswept)
    return sizes, frac, st


# ---------------------------------------------------------------- the benchmark's shape


@pytest.mark.parametrize("pen", [1, 0])
def test_cfg2_at_the_benchmark_shape(pkg, M, pen):
    from test_gpu_matcher_prune_lists import cfg2_inputs
    B = 1024
    params, laser, ranges, poses, bran, bpos, sensor = cfg2_inputs(pkg, range(1_000_000, 1_000_000 + B))
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, pen, 0)
    m = M.ScanMatcher(params, laser, max_batch=B, max_base_scans=1)
    m.set_scans(ranges, poses)
    m.add_scans(bran, bpos)
    sample = set(np.random.default_rng(7 + pen).choice(B, SAMPLE, replace=False).tolist())

    def ctx(b):
        pm = port.PortMatcher(params, laser)
        pm.set_scan(ranges[b], poses[b])
        pm.add_scans(bran[b], bpos[b])
        gx, gy = kv.lattice(pm.sp, pm.grid_off, se, pm.g, 0.05)
        assert np.array_equal(m.grid(b)[0], pm.grid)
        return Ctx(pm.grid, pm.g, pm.compute_offsets(pm.sp[2], se.angle_offset, se.angle_res),
                   int(gx[0, 0] + gy[0, 0] * pm.g.width_step), pm.pts, pm.sp, pm.grid_off, pm.sp[2])

    sizes, frac, _ = check_pruned(m, sensor, se, laser.n_readings, params, ctx, sample)
    m.close()
    assert len(sizes) == SAMPLE
    if pen:
        assert frac >= 0.6, frac


# ---------------------------------------------------------------- round (c) past the accumulator rows


def round_c_batch():
    """uniform grids of 100 with the distance penalty off and an angle penalty whose floor (0.85) lies below the cut
    (L - 0.1 = 0.9): every angle within 0.707 w of the centre reaches the cut, so round (c) grows with w.  (w, angle
    offset, angle step) in degrees, picked with the numpy rounds: 161 angles at w = 8 and 16, and 51 and 52 angles
    (the last group of 3, and of 4) all reaching the cut at w = 40.  -> [(batch, search)]"""
    from test_gpu_matcher_prune_tail import batch
    out = []
    for w, off, res in ROUND_C:
        bt = batch(1081, 1, 830 + int(10 * w + off), minimum_distance_penalty=1.0, minimum_angle_penalty=0.85,
                   angle_variance_penalty=(w * D) ** 2)
        bt.grids[:] = 100
        out.append((bt, kv.window_search(bt, angle_offset=off * D, angle_res=res * D)))
    return out


ROUND_C = [(8.0, 20, 0.25), (16.0, 20, 0.25), (40.0, 12.5, 0.5), (40.0, 12.75, 0.5)]


def round_sizes_of(cases):
    from test_gpu_matcher_prune_bound_items import round_sizes
    return [s for bt, se in cases for s in round_sizes(bt, se)]


def test_round_c_past_the_accumulator_rows(M):
    cases = round_c_batch()
    want = [s[2] for s in round_sizes_of(cases)]
    got = []
    for bt, se in cases:
        m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
        m.set_scans(bt.ranges, bt.poses)
        m.set_grids(bt.grids, bt.offs)
        sizes, _, _ = check_pruned(m, bt.centers, se, bt.laser_s.n_readings, bt.params, batch_ctx(bt, se),
                                   sample=range(bt.B))
        m.close()
        got += [len(sizes[b]["round_c"]) for b in range(bt.B)]
    assert got == want
    assert any(17 <= v < 31 for v in got) and 31 in got and 32 in got and any(v > 64 for v in got), got


# ---------------------------------------------------------------- the fp32 brackets' edges


BRACKET_RES = [1.0, 0.05, 0.002]  # degrees: spreads of a few cells near the sensor / far points / the cut-off


def bracket_batch(angle_res_deg=1.0, B=8):
    """1081 beams: 40 % within 9 m, 10 % at 9 - 12 m (windows across the grid's edges), 20 % at 15 - 30 m (corners
    wholly outside, on every side), 25 % at 405 - 415 m (8192 cells at 0.05 m: 409.6 m), NaN / inf dropouts; half the
    matches 1e5 m from the origin; walls and the scan's own cells on the grid"""
    rng = np.random.default_rng(950 + int(angle_res_deg * 1000))
    params = abi.matcher_params(*kv.SMALL)
    laser_s = synth.Laser(n_readings=1081, min_angle=synth.deg2rad(-135), angular_resolution=synth.deg2rad(0.25),
                          range_threshold=9.25, max_range=1000.0)
    n = laser_s.n_readings
    band = rng.choice(4, size=(B, n), p=[0.45, 0.1, 0.2, 0.25])
    lo, hi = np.array([0.3, 9.0, 15.0, 405.0]), np.array([9.0, 12.0, 30.0, 415.0])
    ranges = rng.uniform(lo[band], hi[band])
    drop = rng.random((B, n)) < 0.03
    ranges[drop] = np.where(rng.random(drop.sum()) < 0.5, np.nan, np.inf)
    poses = np.column_stack([rng.uniform(-2, 2, B), rng.uniform(-2, 2, B), rng.uniform(-math.pi, math.pi, B)])
    poses[B // 2:, :2] += [1e5, -1e5]
    bt = kv.Batch(params, laser_s, ranges, poses)
    se = kv.window_search(bt, angle_offset=20 * angle_res_deg * D, angle_res=angle_res_deg * D)
    from test_gpu_matcher_prune_planes import scan_cells
    scan_cells(bt, se)
    walls(bt, np.random.default_rng(951))
    return bt, se


def bracket_edges(bt, se):
    """how many (group, beam) pairs of the regular matches reach each edge"""
    na = abi.n_steps(se.angle_offset, se.angle_res)
    out = dict.fromkeys(["spread3", "spread4", "near_tie", "cutoff", "nonfinite", "class4", "class255_before",
                         "class255_after", "far_offset"], 0)
    ctx = batch_ctx(bt, se)
    for b in range(bt.B):
        c = ctx(b)
        if c is None:
            continue
        br = gr.Brackets(c.lx, c.ly, c.ch, se.angle_offset, se.angle_res, na, c.gox, c.goy, 1.0 / bt.resolution)
        vx, vy, _, _ = gr.exact_values(c.lx, c.ly, c.ch, se.angle_offset, se.angle_res, na, c.gox, c.goy,
                                       1.0 / bt.resolution)
        sp = np.maximum(br.Mx - br.mx, br.My - br.my)
        out["spread3"] += int((br.inside & (sp == 3)).sum())
        out["spread4"] += int((br.inside & (sp == 4)).sum())
        with np.errstate(invalid="ignore"):
            tie = (np.abs(np.abs(vx - np.floor(vx)) - 0.5) < 1e-4) | (np.abs(np.abs(vy - np.floor(vy)) - 0.5) < 1e-4)
        out["near_tie"] += int(tie[br.members].any(axis=1)[br.corner].sum())
        # past the cut-off, but with brackets that would otherwise take the corner: the 8192 test alone decides
        ends = np.maximum.reduce([np.abs(e.astype(np.float64)) for e in (br.xl, br.xh, br.yl, br.yh)])
        with np.errstate(invalid="ignore"):
            sp_all = np.maximum(np.floor(br.xh + 0.5) - np.ceil(br.xl - 0.5), np.floor(br.yh + 0.5) - np.ceil(br.yl - 0.5))
        out["cutoff"] += int(((ends >= 8192) & (ends < 8300) & (sp_all <= 3)).sum())
        out["nonfinite"] += int((~np.isfinite(c.lx)).sum())
        a, cls = br.corner_class(c.base00, bt.g.width_step, 8 * bt.g.width_step, bt.g.data_size)
        out["class4"] += int((cls == 4).sum())
        # the class is a flat-index test: wholly before the grid's first byte, or wholly past its last
        out["class255_before"] += int(((cls == 255) & (a < 0)).sum())
        out["class255_after"] += int(((cls == 255) & (a >= bt.g.data_size)).sum())
        out["far_offset"] += int(abs(c.gox) > 1e4)
    return out


@pytest.mark.parametrize("angle_res_deg", BRACKET_RES)
def test_bracket_edges(M, angle_res_deg):
    bt, se = bracket_batch(angle_res_deg)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    sizes, _, st = check_pruned(m, bt.centers, se, bt.laser_s.n_readings, bt.params, batch_ctx(bt, se),
                                sample=range(bt.B))
    m.close()
    assert len(sizes) == int((~np.isnan(st["cut"])).sum()) >= bt.B - 2, len(sizes)  # deep-checked matches


# ---------------------------------------------------------------- bounds attained, the cut's edge


def test_grids_of_uniform_blocks(M):
    """grids of 4 x 4 and 7 x 7-aligned blocks of one value each, 3 beams, penalty off: where a beam's window origins
    are block-aligned the pooled image equals the grid at the bound's corners, and the bound of an angle equals its
    best exact response; every match has such angles"""
    bt, _ = kv.uniform_batch(3, 0, B=4)
    ws = bt.g.width_step
    for b in range(bt.B):
        k = 4 if b % 2 == 0 else 7
        rng = np.random.default_rng(960 + b)
        cells = rng.integers(20, 101, size=((bt.g.height + k - 1) // k, (ws + k - 1) // k))
        bt.grids[b] = np.kron(cells, np.ones((k, k), dtype=np.int64))[:bt.g.height, :ws].ravel()
    se = kv.window_search(bt, angle_offset=10 * D, angle_res=0.5 * D, pen=0)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    sizes, _, _ = check_pruned(m, bt.centers, se, bt.laser_s.n_readings, bt.params, batch_ctx(bt, se),
                               sample=range(bt.B))
    m.close()
    assert len(sizes) == bt.B
    for b, d in sizes.items():
        assert (d["ubr"] == d["best"]).any(), b  # the bound attained


CUT = (1.0 - 0.1) - 1e-9  # k_prune_select's cut when the probe's best response L is 1


def cut_edge_batch(floor):
    """every byte 100, the distance penalty off, 1081 beams: every candidate of angle k sums 100 N, so its response
    and its bound are both apen(k) and L = 1.  The angle penalty falls to its floor `floor` 5.7 degrees off the centre
    (w = 8 degrees, 81 angles over +-20): the far angles' bounds are exactly `floor`, and most of them are bounded in
    round (c) (k_sweep_bound<., BOUND_SELECT>), which keeps an angle iff its bound >= the cut"""
    from test_gpu_matcher_prune_tail import batch
    bt = batch(1081, 2, 990, minimum_distance_penalty=1.0, minimum_angle_penalty=floor,
               angle_variance_penalty=(8 * D) ** 2)
    bt.grids[:] = 100
    return bt, kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)


CUT_EDGES = {"at_L_minus_0.1": 0.9, "at_the_cut": CUT, "one_unit_below": float(np.nextafter(CUT, 0.0))}


@pytest.mark.parametrize("edge", list(CUT_EDGES))
def test_bound_at_the_cut(M, edge):
    """round (c) angles whose bound is L - 0.1 (above the cut by its 1e-9), exactly the cut (kept: the selection is
    >=), and one unit in the last place below it (left out); each bound equals its angle's best exact response"""
    floor = CUT_EDGES[edge]
    bt, se = cut_edge_batch(floor)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    sizes, _, st = check_pruned(m, bt.centers, se, bt.laser_s.n_readings, bt.params, batch_ctx(bt, se),
                                sample=range(bt.B))
    m.close()
    assert len(sizes) == bt.B
    for b, d in sizes.items():
        assert st["cut"][b] == CUT
        assert np.array_equal(d["ubr"], d["best"])  # every bound attained
        c = np.array(d["round_c"], dtype=np.int64)
        at_floor = c[st["ubr"][b][c] == floor]  # round (c) angles bounded on the device at the floor
        assert len(at_floor) > 0, b
        assert st["swept"][b][at_floor].all() == (floor >= CUT) and st["swept"][b][at_floor].any() == (floor >= CUT)


# ---------------------------------------------------------------- a generic-kernel match among pruned ones


def test_irregular_lattice_among_pruned_matches(M):
    bt, se0 = kv.irregular_batch(1, seed=970, B=6)
    se = abi.Search(se0.offset_x, se0.offset_y, se0.res_x, se0.res_y, 20 * D, 1 * D, 1, 0)
    bt.centers[0] = kv.rounding_tie_center(bt, 0, se)
    from test_gpu_matcher_prune_planes import scan_cells
    scan_cells(bt, se)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    _, frac, st = check_pruned(m, bt.centers, se, bt.laser_s.n_readings, bt.params, batch_ctx(bt, se),
                               sample=range(bt.B))
    m.close()
    assert math.isnan(st["cut"][0]) and st["swept"][0].all() and np.isnan(st["ubr"][0]).all()
    assert frac > 0.0 and not np.isnan(st["cut"][2:]).any()


def test_read_back_refuses_stale_or_mis_sized_state(pkg, M):
    """the state is sized by the library from the last sweep (8 matches), and refused once set_scans replaced that
    sweep's inputs (here with 4 matches) or response_sums re-swept it; arrays sized for another shape are refused
    before anything is written"""
    import ctypes as C
    from test_gpu_matcher_prune_lists import cfg2_inputs
    A = cfg2_inputs(pkg, range(1_000_000, 1_000_008))
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m = M.ScanMatcher(A[0], A[1], max_batch=8, max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    m.correlate_scan(A[6], se)
    st = m.last_prune_state()
    assert st["ubr"].shape == (8, 181) and st["gub"].shape == (8, 46) and st["cut"].shape == (8,)
    dims = np.array([4, 181], dtype=np.int32)
    small = np.full((4, 181), 7.0)
    rc = m.L.b2s_matcher_last_prune_state(m.h, dims.ctypes.data_as(C.POINTER(C.c_int32)),
                                          small.ctypes.data_as(C.POINTER(C.c_double)), None, None, None)
    assert rc == abi.B2S_ERR_BAD_PARAMS and list(dims) == [8, 181] and (small == 7.0).all()
    m.set_scans(A[2][:4], A[3][:4])
    with pytest.raises(M.B2SError) as e:
        m.last_prune_state()
    assert e.value.status == abi.B2S_ERR_BAD_STATE
    m.add_scans(A[4][:4], A[5][:4])
    m.correlate_scan(A[6][:4], se)
    assert m.last_prune_state()["ubr"].shape == (4, 181)
    m.response_sums(0, (31, 31, 181))
    with pytest.raises(M.B2SError) as e:
        m.last_prune_state()
    assert e.value.status == abi.B2S_ERR_BAD_STATE
    m.close()
