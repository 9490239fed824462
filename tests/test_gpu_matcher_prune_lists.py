"""The window lists of a pruned correlative sweep (csrc/karto_matcher.cu): k_sweep_bound places every beam itself and
k_offsets_sorted lists only the angles the probe and the selection sweep.  On the device:

- lists left over from an earlier search on the same handle never stand in for a selected angle's lists;
- the response volume read back after a pruned call is the whole volume (the skipped angles are listed and swept then);
- the bound drops exactly the beams the lists drop: the pruned fraction equals a numpy restatement of the bound over the
  beams that are neither outside the grid nor over empty 4 x 4 blocks, and the empty-window fraction equals the
  restatement's count of the latter over every (beam, angle) pair."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_prune_bound import INVALID, angle_bounds, kept_angles, responses, synth_case, walls

pytestmark = pytest.mark.gpu
TOL = 1e-9
SEEDS_A = range(1_000_000, 1_000_006)
SEEDS_B = range(2_000_000, 2_000_006)


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def cfg2_inputs(pkg, seeds):
    from oracle import port
    synth = pkg.synth
    params, laser = abi.matcher_params(1.5, 0.05, 0.03, 9.25), abi.laser_from(synth.Laser())
    cases = [synth.make_match_case(s, synth.Laser(), dropout=0.02 if s % 4 == 3 else 0.0) for s in seeds]
    ranges, poses = np.stack([c.ranges for c in cases]), np.stack([c.odom_pose for c in cases])
    bran, bpos = np.stack([c.base_ranges for c in cases])[:, None, :], np.stack([c.base_pose for c in cases])[:, None, :]
    sensor = np.stack([port.PortMatcher(params, laser).sensor_pose(p) for p in poses])
    return params, laser, ranges, poses, bran, bpos, sensor


def restatement(params, laser, ranges, poses, bran, bpos, se, b):
    from oracle import port
    pm = port.PortMatcher(params, laser)
    pm.set_scan(ranges[b], poses[b])
    pm.add_scans(bran[b], bpos[b])
    rc, res = pm.correlate_scan(pm.sp, se, want_sums=True)
    return rc, res, pm.last_sums


def assert_matches_restatement(gpu, b, rc, res):
    resp, pose, cov, status, ties = gpu
    assert status[b] == rc, (b, status[b], rc)
    if rc:
        return
    assert abs(resp[b] - res.response) <= TOL, b
    assert np.allclose(pose[b], res.pose[:], rtol=0, atol=TOL), b
    assert np.allclose(cov[b].ravel(), res.cov[:], rtol=0, atol=TOL), b
    assert ties[b] == res.tie_count, (b, ties[b], res.tie_count)


@pytest.mark.parametrize("pen", [1, 0])
def test_lists_of_an_earlier_search_are_not_reused(pkg, M, pen):
    """a pruned search on scans and grids A, then one on B on the same handle: B's results equal a dense sweep of B
    byte for byte and the restatement within 1e-9"""
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, pen, 0)
    A, Bi = cfg2_inputs(pkg, SEEDS_A), cfg2_inputs(pkg, SEEDS_B)
    params, laser = A[0], A[1]
    m = M.ScanMatcher(params, laser, max_batch=len(SEEDS_A), max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    m.correlate_scan(A[6], se)
    assert m.last_pruned_frac() > 0 or not pen
    m.set_scans(Bi[2], Bi[3])
    m.add_scans(Bi[4], Bi[5])
    pruned = m.correlate_scan(Bi[6], se)
    frac = m.last_pruned_frac()
    m.set_kernel(3)
    dense = m.correlate_scan(Bi[6], se)
    m.set_kernel(0)
    for p, d in zip(pruned, dense):
        assert p.tobytes() == d.tobytes()
    if pen:
        assert frac >= 0.6, frac
    for b in range(len(SEEDS_B)):
        rc, res, _ = restatement(*Bi[:6], se, b)
        assert_matches_restatement(pruned, b, rc, res)
    m.close()


def test_read_back_after_pruning_cfg2(pkg, M):
    """response_sums right after a pruned call (after a different search on the same handle): the whole volume"""
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    A, Bi = cfg2_inputs(pkg, SEEDS_A[:4]), cfg2_inputs(pkg, SEEDS_B[:4])
    m = M.ScanMatcher(A[0], A[1], max_batch=4, max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    m.correlate_scan(A[6], se)
    m.set_scans(Bi[2], Bi[3])
    m.add_scans(Bi[4], Bi[5])
    m.correlate_scan(Bi[6], se)
    assert m.last_pruned_frac() >= 0.6
    for b in range(4):
        rc, _, sums = restatement(*Bi[:6], se, b)
        assert rc == 0
        assert np.array_equal(m.response_sums(b, (31, 31, 181)), sums), b
    m.close()


@pytest.mark.parametrize("pen", [1, 0])
def test_read_back_after_pruning_walls(M, pen):
    """crafted grids with walls along every edge and across row ends (edge beams, row-wrap beams: the bound's
    checked path): the volume read back after a pruned call is the restatement's and the brute-force sum's"""
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=510, B=16)
    walls(bt, np.random.default_rng(511))
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D, pen=pen)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu = m.correlate_scan(bt.centers, se)
    assert m.last_timing()["path"] == 2
    dims = (abi.n_steps(se.offset_y, se.res_y), abi.n_steps(se.offset_x, se.res_x), 41)
    for b in range(bt.B):
        rc, res, sums = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)
        if rc == 0:
            vol = m.response_sums(b, dims)
            assert np.array_equal(vol, sums), b
            if b % 4 == 0:
                assert np.array_equal(vol, bt.brute(b, se)), b
    m.close()


def dropped_beams(grid, g, lut, base00, nx, ny):
    """[na][n]: (the beam's window is dropped from the lists, it is dropped as an empty window), as k_offsets_sorted
    classifies a stride-1 single-tile search: not finite, wholly outside [0, data_size), or - when it does not wrap a
    row end - covering only 4 x 4 blocks without a non-zero cell"""
    ws, ds, h = g.width_step, g.data_size, g.height
    valid = lut != INVALID
    a = ((base00 + lut.astype(np.int64) + 2**31) % 2**32) - 2**31  # int32 arithmetic of base + offset
    ac = np.clip(a, -(1 << 29), 1 << 29)
    span = min(31 * ws + 32 + 8, 1 << 29)  # 32 candidate rows, a 32-byte tile row, 8 bytes of alignment
    outside = (ac + span < 0) | (ac - 8 >= ds)
    sbx, sby = (ws + 3) // 4, (h + 3) // 4
    img = np.zeros((sby * 4, sbx * 4), dtype=np.int64)
    img[:h, :ws] = grid.reshape(h, ws)
    nonempty = img.reshape(sby, 4, sbx, 4).max(axis=(1, 3)) > 0
    sat = np.zeros((sby + 1, sbx + 1), dtype=np.int64)
    sat[1:, 1:] = nonempty.cumsum(axis=0).cumsum(axis=1)
    y = np.floor_divide(a, ws)
    x = a - y * ws
    test = valid & ~outside & (a >= 0) & (x + nx <= ws) & (y + ny <= h)
    bx0, bx1 = np.clip(x >> 2, 0, sbx - 1), np.clip((x + nx - 1) >> 2, 0, sbx - 1)
    by0, by1 = np.clip(y >> 2, 0, sby - 1), np.clip((y + ny - 1) >> 2, 0, sby - 1)
    cnt = sat[by1 + 1, bx1 + 1] - sat[by0, bx1 + 1] - sat[by1 + 1, bx0] + sat[by0, bx0]
    empty = test & (cnt == 0)
    return ~valid | outside | empty, empty


def test_pruned_and_empty_fractions_against_a_restatement(pkg, M):
    """last_pruned_frac(): the numpy bound over the beams the lists keep, k_prune_probe's and k_prune_select's rule on
    the restatement's exact volume; empty_window_frac: the restatement's empty windows over every (beam, angle)"""
    seeds = list(range(1_000_000, 1_000_004))
    A = cfg2_inputs(pkg, seeds)
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m = M.ScanMatcher(A[0], A[1], max_batch=len(seeds), max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    out = m.correlate_scan(A[6], se)
    assert (out[3] == 0).all()
    frac, empty_frac = m.last_pruned_frac(), m.last_stats()["empty_window_frac"]
    m.close()
    pruned = empties = 0
    for s in seeds:
        grid, g, lut, base00, sums, n, se_, params, ch = synth_case(s, 1)
        drop, empty = dropped_beams(grid, g, lut, base00, 31, 31)
        ubr = angle_bounds(grid, g.width_step, np.where(drop, INVALID, lut), base00, n, se_, params, ch)
        keep = kept_angles(ubr, responses(sums, n, se_, params, ch))
        pruned += int((~keep).sum())
        empties += int(empty.sum())
    na, n = 181, A[1].n_readings
    assert frac == pruned / (float(len(seeds)) * na), (frac, pruned)
    assert empty_frac == empties / (float(len(seeds)) * na * n), (empty_frac, empties)
    assert 0.6 <= frac < 1.0 and empty_frac > 0.0
