"""The upper bound behind the correlative sweep's angle pruning (k_grid_pool, k_sweep_bound, k_prune_probe,
k_prune_select in csrc/karto_matcher.cu), restated in numpy on the C restatement's grids and volumes, without a GPU.

For every case: the bound of each angle is at least every exact response of that angle, and no angle the rule leaves
out holds a candidate whose response reaches best - 0.1 (so the best pose, its ties and every cell maximum the
positional covariance reads are unchanged).  The restatement keeps every beam; the device also leaves out beams whose
whole window is empty, which add 0 to every candidate and so to neither side."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi, port, synth

GAIN = 0.2          # DISTANCE_PENALTY_GAIN, ANGLE_PENALTY_GAIN (Mapper.cpp:37-38)
PROBE = 16          # PRUNE_PROBE
INVALID = np.iinfo(np.int32).max


def pooled(grid, ws):
    """P[f] for f in [-4 ws, data_size): max over dy, dx in [0, 4) of grid[f + dy ws + dx] in flat index space"""
    ds, lead = len(grid), 4 * ws
    ext = np.zeros(lead + ds + 4 * ws + 4, dtype=np.int64)
    ext[lead:lead + ds] = grid
    f = np.arange(-lead, ds)
    return np.max([ext[lead + f + dy * ws + dx] for dy in range(4) for dx in range(4)], axis=0)


def responses(sums, n, se, params, center_h):
    """candidate_response of every candidate of an int volume [ny][nx][na], in its operation order"""
    ny, nx, na = sums.shape
    x = -se.offset_x + np.arange(nx, dtype=np.float64) * se.res_x
    y = -se.offset_y + np.arange(ny, dtype=np.float64) * se.res_y
    sq = (x[None, :] * x[None, :] + y[:, None] * y[:, None])[:, :, None]
    angle = (center_h - se.angle_offset) + np.arange(na, dtype=np.float64) * se.angle_res
    r = sums.astype(np.float64) / float(n * 100)
    if not se.do_penalize:
        return r
    dpen = np.maximum(1.0 - (GAIN * sq / params.distance_variance_penalty), params.minimum_distance_penalty)
    sq_a = (angle - center_h) * (angle - center_h)
    apen = np.maximum(1.0 - (GAIN * sq_a / params.angle_variance_penalty), params.minimum_angle_penalty)
    return np.where(np.abs(r) < 1e-6, r, r * (dpen * apen[None, None, :]))


def angle_bounds(grid, ws, lut, base00, n, se, params, center_h):
    """UBr(k): the largest block bound of angle k, 8 x 8 blocks of 4 x 4 candidates (k_sweep_bound)"""
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    assert nx <= 32 and ny <= 32
    P, lead, ds = pooled(grid, ws), 4 * ws, len(grid)
    na = lut.shape[0]
    u = np.zeros((na, 8, 8), dtype=np.int64)
    for by in range(8):
        for bx in range(8):
            # flat index of the block corner, modulo 2^32 as the reference's base + offset
            f = ((base00 + lut.astype(np.int64) + 4 * by * ws + 4 * bx + 2**31) % 2**32) - 2**31
            inside = (lut != INVALID) & (f >= -lead) & (f < ds)
            u[:, by, bx] = np.where(inside, P[np.clip(f + lead, 0, len(P) - 1)], 0).sum(axis=1)
    # every candidate gets its block's sum and its block's largest distance penalty: the bound of the block
    sums = np.repeat(np.repeat(u.transpose(1, 2, 0), 4, axis=0), 4, axis=1)[:ny, :nx]
    r = sums / float(n * 100)
    if se.do_penalize:  # also below 1e-6, where the reference does not penalise: the selection rule covers that band
        r = r * penalties(se, params, center_h, nx, ny, na)
    return r.reshape(-1, na).max(axis=0)


def penalties(se, params, center_h, nx, ny, na):
    """dpen * apen of every candidate, dpen the largest distance penalty of the candidate's 4 x 4 block"""
    x = -se.offset_x + np.arange(nx, dtype=np.float64) * se.res_x
    y = -se.offset_y + np.arange(ny, dtype=np.float64) * se.res_y
    dpen = np.maximum(1.0 - (GAIN * (x[None, :] * x[None, :] + y[:, None] * y[:, None]) / params.distance_variance_penalty),
                      params.minimum_distance_penalty)
    pad = np.full((32, 32), -np.inf)
    pad[:ny, :nx] = dpen
    dpen = np.repeat(np.repeat(pad.reshape(8, 4, 8, 4).max(axis=(1, 3)), 4, axis=0), 4, axis=1)[:ny, :nx]
    angle = (center_h - se.angle_offset) + np.arange(na, dtype=np.float64) * se.angle_res
    apen = np.maximum(1.0 - (GAIN * ((angle - center_h) * (angle - center_h)) / params.angle_variance_penalty),
                      params.minimum_angle_penalty)
    return dpen[:, :, None] * apen[None, None, :]


def walls(bt, rng):
    """dense walls along the grid's edges, across row ends (flat-index wrap) and through the middle, on top of
    probe_batch's isolated cells: responses high enough that pruning has work to do, at every edge a window can reach"""
    g = bt.g
    ws, h = g.width_step, g.height
    for b in range(bt.B):
        img = bt.grids[b].reshape(h, ws)
        v = lambda shape: rng.integers(40, 101, size=shape)  # noqa: E731
        img[:3, :] = v((3, ws))                      # first rows
        img[-3:, :] = v((3, ws))                     # last rows
        img[:, :2] = v((h, 2))                       # first columns: neighbours of the previous row's end
        img[:, g.width - 2:] = v((h, ws - g.width + 2))  # last columns and padding
        r = int(rng.integers(h // 4, 3 * h // 4))
        img[r:r + 2, :] = v((2, ws))                 # a wall through the search window's rows
        c = int(rng.integers(ws // 4, 3 * ws // 4))
        img[:, c:c + 2] = v((h, 2))


def kept_angles(ubr, resp):
    """k_prune_probe + k_prune_select: the PROBE largest bounds swept exactly; L their best; keep UBr >= L - 0.1 - 1e-9"""
    na = len(ubr)
    order = sorted(range(na), key=lambda k: (-ubr[k], k))
    probe = np.zeros(na, dtype=bool)
    probe[order[:min(PROBE, na)]] = True
    L = resp[:, :, probe].max()
    if not (L - 0.1 > 1e-6):
        return np.ones(na, dtype=bool)
    return probe | (ubr >= L - 0.1 - 1e-9)


def check_case(grid, g, lut, base00, sums, n, se, params, center_h):
    resp = responses(sums, n, se, params, center_h)
    ubr = angle_bounds(grid, g.width_step, lut, base00, n, se, params, center_h)
    per_angle = resp.reshape(-1, resp.shape[2]).max(axis=0)
    assert (ubr >= per_angle).all(), np.flatnonzero(ubr < per_angle)
    keep = kept_angles(ubr, resp)
    best = resp.max()
    assert (per_angle[~keep] < best - 0.1).all()
    return 1.0 - keep.mean()


def synth_case(seed, pen):
    params, laser = abi.matcher_params(1.5, 0.05, 0.03, 9.25), abi.laser_from(synth.Laser())
    c = synth.make_match_case(seed, synth.Laser(), dropout=0.02 if seed % 4 == 3 else 0.0)
    pm = port.PortMatcher(params, laser)
    pm.set_scan(c.ranges, c.odom_pose)
    pm.add_scans(c.base_ranges[None, :], c.base_pose[None, :])
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, pen, 0)
    rc, _ = pm.correlate_scan(pm.sp, se, want_sums=True)
    assert rc == 0
    gx, gy = kv.lattice(pm.sp, pm.grid_off, se, pm.g, 0.05)
    base00 = int(gx[0, 0] + gy[0, 0] * pm.g.width_step)
    lut = pm.compute_offsets(pm.sp[2], se.angle_offset, se.angle_res)
    return pm.grid, pm.g, lut, base00, pm.last_sums, laser.n_readings, se, params, pm.sp[2]


@pytest.mark.parametrize("pen", [1, 0])
def test_cfg2_matches(pen):
    fracs = [check_case(*synth_case(s, pen)) for s in range(1_000_000, 1_000_004)]
    if pen:
        assert np.mean(fracs) >= 0.6, fracs


def batch_cases(bt, se):
    for b in range(bt.B):
        rc, _, sums = bt.oracle(b, se)
        if rc:
            continue
        gx, gy = bt.cells(b, se)
        if not kv.is_regular(gx, gy, 1):
            continue
        yield (bt.grids[b], bt.g, bt.lut(b, se), int(gx[0, 0] + gy[0, 0] * bt.g.width_step), sums,
               bt.laser_s.n_readings, se, bt.params, bt.centers[b][2])


@pytest.mark.parametrize("pen", [1, 0])
def test_walls_at_grid_edges_and_row_ends(pen):
    """probe_batch's isolated cells (window corners, block edges, padding, both ends of the data, row ends) plus walls
    along every edge of the grid and across row ends: windows that leave the grid and wrap a row end"""
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=500, B=8)
    walls(bt, np.random.default_rng(501))
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D, pen=pen)
    fracs = [check_case(*c) for c in batch_cases(bt, se)]
    assert len(fracs) >= 6


def test_best_below_the_margin_keeps_every_angle():
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=502, B=4)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    for c in batch_cases(bt, se):
        assert check_case(*c) == 0.0


@pytest.mark.parametrize("pen", [1, 0])
def test_uniform_room_all_candidates_near_the_best(pen):
    """every byte 100: every candidate of an angle ties; without the penalty nothing may be left out"""
    bt, _ = kv.uniform_batch(1081, 100, B=2)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D, pen=pen)
    fracs = [check_case(*c) for c in batch_cases(bt, se)]
    assert len(fracs) == 2 and (pen or max(fracs) == 0.0)
