"""The group pass of the correlative sweep's angle pruning (k_grid_pool<7>, k_sweep_bound<., BOUND_GROUPS> and the
three bound rounds of k_sweep_bound<., BOUND_PROBE>, k_prune_select and k_sweep_bound<., BOUND_SELECT> in
csrc/karto_matcher.cu), restated in numpy on the C restatement's grids and volumes, without a GPU.

For every case: the bound of a group of BOUND_GROUP consecutive angles, read from the 7 x 7 pooled image at the low
corner of each beam's origins (or, when they spread more than 3 cells on an axis, the largest over the members'
origins), is at least the single-angle bound UBr of every member; and bounding single angles only in the groups the
rounds pick gives exactly the probe and kept sets of bounding every angle, ties included."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D
from test_prune_bound import (INVALID, PROBE, angle_bounds, batch_cases, kept_angles, penalties, responses, synth_case,
                              walls)

GROUP = 4   # BOUND_GROUP
SPREAD = 3  # BOUND_SPREAD


def pooled7(grid, ws):
    """P7[f] for f in [-8 ws, data_size): max over dy, dx in [0, 7) of grid[f + dy ws + dx] in flat index space"""
    ds, lead = len(grid), 8 * ws
    ext = np.zeros(lead + ds + 7 * ws + 7, dtype=np.int64)
    ext[lead:lead + ds] = grid
    f = np.arange(-lead, ds)
    return np.max([ext[lead + f + dy * ws + dx] for dy in range(7) for dx in range(7)], axis=0)


def group_bounds(grid, ws, lut, base00, n, se, params, center_h, stats=None):
    """gub[g]: the largest block bound of group g from P7 (k_sweep_bound<., BOUND_GROUPS>)"""
    nx, ny = kv_steps(se)
    P7, lead, ds = pooled7(grid, ws), 8 * ws, len(grid)
    na, nb = lut.shape
    ng = (na + GROUP - 1) // GROUP
    valid = lut != INVALID
    l64 = lut.astype(np.int64)
    gy = np.where(valid, np.floor((l64 + ws // 2) / ws), 0).astype(np.int64)  # lookup values are within ws / 2 cells
    gx = np.where(valid, l64 - gy * ws, 0)
    u = np.zeros((ng, 8, 8), dtype=np.int64)
    big = np.iinfo(np.int64).max // 4

    def P7_at(f):
        f = ((f + 2**31) % 2**32) - 2**31
        return np.where((f >= -lead) & (f < ds), P7[np.clip(f + lead, 0, len(P7) - 1)], 0)

    for g in range(ng):
        ks = range(g * GROUP, min(g * GROUP + GROUP, na))
        v = valid[ks]
        mx = np.where(v, gx[ks], big).min(axis=0)
        my = np.where(v, gy[ks], big).min(axis=0)
        sx = np.where(v, gx[ks], -big).max(axis=0) - mx
        sy = np.where(v, gy[ks], -big).max(axis=0) - my
        corner = v.all(axis=0) & (sx <= SPREAD) & (sy <= SPREAD)
        if stats is not None:
            stats["fallback"] = stats.get("fallback", 0) + int((~corner & v.any(axis=0)).sum())
        for by in range(8):
            for bx in range(8):
                off = 4 * by * ws + 4 * bx
                at_corner = P7_at(base00 + mx + my * ws + off)
                members = np.where(v, P7_at(base00 + l64[ks] + off), 0).max(axis=0)
                u[g, by, bx] = np.where(corner, at_corner, np.where(v.any(axis=0), members, 0)).sum()
    sums = np.repeat(np.repeat(u.transpose(1, 2, 0), 4, axis=0), 4, axis=1)[:ny, :nx]
    r = sums / float(n * 100)
    if se.do_penalize:
        pen = penalties(se, params, center_h, nx, ny, na)
        r = r * np.stack([pen[:, :, g * GROUP:g * GROUP + GROUP].max(axis=2) for g in range(ng)], axis=2)
    return r.reshape(-1, ng).max(axis=0)


def kv_steps(se):
    from karto_volume_reference import abi
    return abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)


def rounds(ubr, gub, resp):
    """rounds (a) - (c): (probe set, kept set, angles bounded one by one), reading ubr only where a round bounds it"""
    na, ng = len(ubr), len(gub)
    T = min(PROBE, na)
    members = [list(range(g * GROUP, min(g * GROUP + GROUP, na))) for g in range(ng)]
    order = sorted(range(ng), key=lambda g: (-gub[g], g))
    ev, top = [], 0
    while len(ev) < T:  # (a)
        ev += members[order[top]]
        top += 1
    f16 = sorted((ubr[k] for k in ev), reverse=True)[T - 1]
    ev += [k for g in order[top:] if gub[g] >= f16 for k in members[g]]  # (b)
    probe = np.zeros(na, dtype=bool)
    probe[sorted(ev, key=lambda k: (-ubr[k], k))[:T]] = True
    L = resp[:, :, probe].max()
    if not (L - 0.1 > 1e-6):
        return probe, np.ones(na, dtype=bool), set(ev)
    cut = L - 0.1 - 1e-9
    evs = set(ev)
    ev_c = [k for k in range(na) if k not in evs and not probe[k] and gub[k // GROUP] >= cut]  # (c)
    evs |= set(ev_c)
    keep = probe | np.array([k in evs and ubr[k] >= cut for k in range(na)])
    return probe, keep, evs


def check_case(grid, g, lut, base00, sums, n, se, params, center_h, stats=None):
    resp = responses(sums, n, se, params, center_h)
    ubr = angle_bounds(grid, g.width_step, lut, base00, n, se, params, center_h)
    gub = group_bounds(grid, g.width_step, lut, base00, n, se, params, center_h, stats)
    na = len(ubr)
    for k in range(na):
        assert gub[k // GROUP] >= ubr[k], (k, gub[k // GROUP], ubr[k])
    probe, keep, evs = rounds(ubr, gub, resp)
    order = sorted(range(na), key=lambda k: (-ubr[k], k))
    assert set(np.flatnonzero(probe)) == set(order[:min(PROBE, na)])
    assert np.array_equal(keep, kept_angles(ubr, resp))
    return len(evs) / na


@pytest.mark.parametrize("pen", [1, 0])
def test_cfg2_matches(pen):
    shares = [check_case(*synth_case(s, pen)) for s in range(1_000_000, 1_000_004)]
    if pen:  # most angles are bounded by their group alone
        assert np.mean(shares) <= 0.4, shares


@pytest.mark.parametrize("pen", [1, 0])
def test_walls_at_grid_edges_and_row_ends(pen):
    """walls along every edge of the grid and across row ends, 1 degree steps: windows that leave the grid and wrap a
    row end, and beams whose origins spread past 3 cells across a group (the per-member fallback)"""
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=500, B=8)
    walls(bt, np.random.default_rng(501))
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D, pen=pen)
    stats = {}
    shares = [check_case(*c, stats=stats) for c in batch_cases(bt, se)]
    assert len(shares) >= 6
    assert stats["fallback"] > 0


def test_best_below_the_margin_keeps_every_angle():
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=502, B=4)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    for c in batch_cases(bt, se):
        check_case(*c)


@pytest.mark.parametrize("pen", [1, 0])
def test_uniform_room_all_candidates_near_the_best(pen):
    bt, _ = kv.uniform_batch(1081, 100, B=2)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D, pen=pen)
    assert len([check_case(*c) for c in batch_cases(bt, se)]) == 2
