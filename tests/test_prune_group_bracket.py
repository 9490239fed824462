"""The fp32 origin brackets of the angle bound's group pass (k_sweep_bound<., BOUND_GROUPS>, restated in
tests/group_bracket_reference.py) contain the exact lookup values of every member angle, without a GPU.

The group pass adds, for a beam whose brackets span at most BOUND_SPREAD cells per axis, P7 at the bracket's low
corner; that covers P at every member's window origin only if kround(((o + gox) - gox) * scale) of every member lies
inside the bracket.  The fp32 margin mg_match + 1e-5 (|px| + |py|) scale is what makes that so; these tests check it
on every (group, beam) of the benchmark's matches and on seeded points at the edges of the margin: grids of 1 mm to
10 cm, grid offsets up to 1e6 m, members within 1e-4 cells of a .5 tie, spreads of exactly 3 and 4 cells and brackets
on both sides of the 8192-cell cut-off.  Each returns the smallest slack (cells between a bracket end and the nearest
unrounded exact value); the smallest over all of them is about 4.0e-3 cells.

The premise tests at the end show that the device cases of tests/test_gpu_matcher_prune_state.py reach the edges they
are named for."""
import math

import numpy as np
import pytest

import group_bracket_reference as gr
from karto_volume_reference import D, abi, port, synth
from test_prune_bound import INVALID, angle_bounds
from test_prune_group_bound import GROUP, SPREAD

MIN_SLACK = 3e-3  # cells: the margin (>= 4e-3) less fp32's rounding of the rotation


def check_points(lx, ly, ch, angle_offset, angle_res, na, gox, goy, scale):
    """every bracket inside 8192 cells contains its members' exact values; -> (smallest slack, Brackets, exact)"""
    br = gr.Brackets(lx, ly, ch, angle_offset, angle_res, na, gox, goy, scale)
    vx, vy, rx, ry = gr.exact_values(lx, ly, ch, angle_offset, angle_res, na, gox, goy, scale)
    finite = np.isfinite(lx) & np.isfinite(ly)
    slack, ok = br.slack(vx, vy, finite)
    assert ok, "a rounded exact lookup value lies outside its fp32 bracket"
    assert slack >= MIN_SLACK, slack
    return slack, br, (vx, vy, rx, ry)


def cfg2_case(seed, pen=1):
    """synth_case of tests/test_prune_bound.py, with the restatement's matcher (for its points and grid offset)"""
    params, laser = abi.matcher_params(1.5, 0.05, 0.03, 9.25), abi.laser_from(synth.Laser())
    c = synth.make_match_case(seed, synth.Laser(), dropout=0.02 if seed % 4 == 3 else 0.0)
    pm = port.PortMatcher(params, laser)
    pm.set_scan(c.ranges, c.odom_pose)
    pm.add_scans(c.base_ranges[None, :], c.base_pose[None, :])
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, pen, 0)
    return pm, se, params, laser


def test_cfg2_every_group_and_beam():
    """every (group, beam) of four benchmark matches (46 groups x 1081 beams, NaN / inf dropouts); the restated
    scan-local points give the restatement's lookup table exactly, and the group bound from the brackets is at least
    the single-angle bound of every member"""
    import karto_volume_reference as kv
    slacks = []
    for s in range(1_000_000, 1_000_004):
        pm, se, params, laser = cfg2_case(s)
        lx, ly = gr.local_points(pm.pts, pm.sp)
        na, scale = abi.n_steps(se.angle_offset, se.angle_res), 1.0 / params.resolution
        lut = pm.compute_offsets(pm.sp[2], se.angle_offset, se.angle_res)
        slack, br, (vx, vy, rx, ry) = check_points(lx, ly, pm.sp[2], se.angle_offset, se.angle_res, na, *pm.grid_off,
                                                   scale)
        with np.errstate(invalid="ignore"):
            ours = np.where(np.isfinite(vx) & np.isfinite(vy),
                            (rx.astype(np.int64) + ry.astype(np.int64) * pm.g.width_step) % 2**32, INVALID)
        assert np.array_equal(ours, lut.astype(np.int64) % 2**32)
        gx, gy = kv.lattice(pm.sp, pm.grid_off, se, pm.g, 0.05)
        base00 = int(gx[0, 0] + gy[0, 0] * pm.g.width_step)
        gub = gr.group_bounds(pm.grid, pm.g, lut, base00, laser.n_readings, se, params, pm.sp[2], br)
        ubr = angle_bounds(pm.grid, pm.g.width_step, lut, base00, laser.n_readings, se, params, pm.sp[2])
        assert (gub[np.arange(na) // GROUP] >= ubr).all()
        slacks.append(slack)
    assert min(slacks) >= MIN_SLACK


@pytest.mark.parametrize("res", [0.001, 0.01, 0.025, 0.05, 0.1])
@pytest.mark.parametrize("angle_res_deg", [0.1, 0.25, 1.0])
def test_seeded_points_out_to_the_range_threshold(res, angle_res_deg):
    """4096 points uniform in a 9.25 m disc (up to 9250 cells at 1 mm: past the cut-off), grid offsets within 50 m"""
    rng = np.random.default_rng(int(res * 1e4) + int(angle_res_deg * 100))
    r, t = 9.25 * np.sqrt(rng.random(4096)), rng.uniform(-math.pi, math.pi, 4096)
    lx, ly = r * np.cos(t), r * np.sin(t)
    gox, goy = rng.uniform(-50, 50, 2)
    check_points(lx, ly, rng.uniform(-math.pi, math.pi), 20 * D, angle_res_deg * D, 41, gox, goy, 1.0 / res)


@pytest.mark.parametrize("gox", [1e3, -1e5, 1e6, -1e6 + 0.37])
def test_far_grid_offsets(gox):
    """the (o + gox) - gox rounding grows with |gox|: mg_match's 1e-15 (|gox| + |goy|) scale term covers it"""
    rng = np.random.default_rng(int(abs(gox)) % 1000)
    lx, ly = rng.uniform(-9, 9, 4096), rng.uniform(-9, 9, 4096)
    check_points(lx, ly, 0.3, 20 * D, 0.25 * D, 161, gox, -0.5 * gox + 0.123, 20.0)


def near_tie_points(n, seed, scale=20.0, gox=3.7, goy=-1.3, k=5, angle_res=0.25 * D, ch=0.4):
    """points whose member k's scaled x coordinate lies within 1e-4 cells of a .5 tie (both sides)"""
    rng = np.random.default_rng(seed)
    a = gr.angles(ch, 20 * D, angle_res, k + 1)[k]
    c, s = math.cos(a), math.sin(a)
    ly = rng.uniform(-8, 8, n)
    v = rng.integers(-150, 150, n) + 0.5 + rng.uniform(-1e-4, 1e-4, n)  # target x in cells
    lx = (v / scale + s * ly) / c
    return lx, ly, ch, 20 * D, angle_res, 41, gox, goy, scale


def test_members_near_a_rounding_tie():
    args = near_tie_points(4096, 3)
    _, br, (vx, _, _, _) = check_points(*args)
    frac = np.abs(np.abs(vx[5] - np.floor(vx[5])) - 0.5)
    assert (frac < 1e-4).mean() > 0.9


def spread_points(n, seed, scale=20.0):
    """1 degree steps out to 9 m: x / y spreads of 0 to ~9 cells across a group"""
    rng = np.random.default_rng(seed)
    r, t = rng.uniform(0.5, 9.0, n), rng.uniform(-math.pi, math.pi, n)
    return r * np.cos(t), r * np.sin(t), 0.1, 20 * D, 1 * D, 41, 2.3, -4.1, scale


def test_spreads_of_three_and_four_cells():
    _, br, _ = check_points(*spread_points(8192, 4))
    sp = np.maximum(br.Mx - br.mx, br.My - br.my)[br.inside]
    assert (sp == SPREAD).sum() > 100 and (sp == SPREAD + 1).sum() > 100
    assert br.corner[br.inside][sp == SPREAD].all() and not br.corner[br.inside][sp == SPREAD + 1].any()


def cutoff_points(n, seed, res=0.001):
    """points 8180 - 8200 cells out on the x axis, 0.01 degree steps: brackets just inside and just outside 8192"""
    rng = np.random.default_rng(seed)
    x = rng.choice([-1, 1], n) * rng.uniform(8180, 8200, n) * res
    return x, rng.uniform(-0.2, 0.2, n), 0.0, 0.2 * D, 0.01 * D, 41, 0.0, 0.0, 1.0 / res


def test_brackets_on_both_sides_of_the_cutoff():
    _, br, _ = check_points(*cutoff_points(4096, 5))
    ends = np.maximum(np.abs(br.xl), np.abs(br.xh))
    assert ((ends < 8192) & (ends > 8191)).any() and ((ends >= 8192) & (ends < 8193)).any()
    assert not br.inside[ends >= 8192].any() and br.corner[ends < 8191].any()


# ---------------------------------------------------------------- premises of the device cases


def test_device_bracket_edge_cases_premise():
    """tests/test_gpu_matcher_prune_state.py bracket_batch: every named edge is reached by some regular match"""
    import test_gpu_matcher_prune_state as st
    got = {}
    for res in st.BRACKET_RES:
        for k, v in st.bracket_edges(*st.bracket_batch(res)).items():
            got[k] = got.get(k, 0) + v
    for name in ("spread3", "spread4", "near_tie", "cutoff", "nonfinite", "class4", "class255_before",
                 "class255_after", "far_offset"):
        assert got[name] > 0, (name, got)


def test_round_c_cases_premise():
    """tests/test_gpu_matcher_prune_state.py round_c_batch: rounds (c) of 17-31, exactly 31, exactly 32 and more than
    64 angles, by the numpy rounds"""
    import test_gpu_matcher_prune_state as st
    sizes = st.round_sizes_of(st.round_c_batch())
    c = [s[2] for s in sizes]
    assert any(17 <= v < 31 for v in c) and 31 in c and 32 in c and any(v > 64 for v in c), sizes


@pytest.mark.parametrize("edge", ["at_L_minus_0.1", "at_the_cut", "one_unit_below"])
def test_cut_edge_cases_premise(edge):
    """tests/test_gpu_matcher_prune_state.py cut_edge_batch: L = 1, so the cut is CUT, and round (c) bounds angles
    whose numpy bound is exactly the penalty floor (L - 0.1, the cut, one unit below it), each kept iff >= the cut"""
    import test_gpu_matcher_prune_state as st
    from test_gpu_matcher_prune_lists import dropped_beams
    from test_prune_bound import batch_cases, responses
    from test_prune_group_bound import group_bounds, rounds
    floor = st.CUT_EDGES[edge]
    bt, se = st.cut_edge_batch(floor)
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    cases = list(batch_cases(bt, se))
    assert len(cases) == bt.B
    for grid, g, lut, base00, sums, n, se_, params, ch in cases:
        drop, _ = dropped_beams(grid, g, lut, base00, nx, ny)
        ubr = angle_bounds(grid, g.width_step, np.where(drop, INVALID, lut), base00, n, se_, params, ch)
        gub = group_bounds(grid, g.width_step, lut, base00, n, se_, params, ch)
        resp = responses(sums, n, se_, params, ch)
        probe, keep, evs = rounds(ubr, gub, resp)
        _, _, ev_ab = rounds(ubr, gub, np.zeros_like(resp))
        assert resp[:, :, probe].max() - 0.1 - 1e-9 == st.CUT
        at_floor = [k for k in evs - ev_ab if ubr[k] == floor]
        assert at_floor and all(keep[k] == (floor >= st.CUT) for k in at_floor), (edge, len(at_floor))
