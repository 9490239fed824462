"""The fp64 tail of a pruned CorrelateScan (csrc/karto_matcher.cu): k_prune_select's L through the float pre-filter,
and k_reduce walking only the angles the pruned sweep swept.  Every case is swept pruned and dense (every beam, every
angle): the results are equal byte for byte and equal the C restatement's, and last_pruned_frac() equals the numpy
restatement of the bound and the selection rule (tests/test_prune_bound.py).

The cases: equal probe sums at many angles under a clamped angle penalty (float near-ties in k_prune_select, at the
maximum and below it) with more than RED_MAX_TIES ties at the best; responses in the 0.5e-6 .. 2e-6 band in which the
pre-filter always evaluates exactly; and cells whose sums are 0 at every swept angle next to cells that are not."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, RED_MAX_TIES, abi
from test_gpu_matcher_prune import assert_matches_restatement, pruned_and_dense
from test_gpu_matcher_prune_lists import dropped_beams
from test_gpu_matcher_prune_planes import scan_cells
from test_prune_bound import INVALID, angle_bounds, batch_cases, kept_angles, responses

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def batch(n, B, seed, **params):
    """B matches of n beams (ranges inside a 4 m grid, no dropouts) with matcher parameters `params`; empty grids"""
    laser_s = kv.make_laser(n, rt=4.0)
    ranges, poses = kv.random_scans(np.random.default_rng(seed), B, laser_s, 0.5, 3.2)
    return kv.Batch(abi.matcher_params(1.5, 0.05, 0.03, 4.0, **params), laser_s, ranges, poses)


def restated_keep(bt, se):
    """the angles the numpy bound and k_prune_select's rule sweep, per match (every match is a regular lattice)"""
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    keep = []
    for grid, g, lut, base00, sums, n, se_, params, ch in batch_cases(bt, se):
        drop, _ = dropped_beams(grid, g, lut, base00, nx, ny)
        ubr = angle_bounds(grid, g.width_step, np.where(drop, INVALID, lut), base00, n, se_, params, ch)
        keep.append(kept_angles(ubr, responses(sums, n, se_, params, ch)))
    assert len(keep) == bt.B
    return keep


def sweep_and_check(M, bt, se):
    """pruned == dense byte for byte, both == the restatement, last_pruned_frac == the numpy rule; -> (results,
    fraction pruned, the restatement's sums of every match, the angles swept of every match)"""
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu, frac = pruned_and_dense(m, bt.centers, se)
    m.close()
    keep = restated_keep(bt, se)
    assert frac == sum(int((~k).sum()) for k in keep) / (float(bt.B) * len(keep[0])), frac
    sums = []
    for b in range(bt.B):
        rc, res, s = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)
        sums.append(s)
    return gpu, frac, sums, keep


def test_clamped_angle_penalty_and_ties_beyond_the_sequential_sum(M):
    """every byte 100, no distance penalty (its minimum is 1) and an angle penalty that reaches its 0.85 floor 1 degree
    off the centre: every candidate of an angle has the same sum, the probe holds the centre, its two neighbours and
    13 angles of equal score at the floor, every other angle is pruned, and the best ties at every cell"""
    bt = batch(1081, 3, 700, minimum_distance_penalty=1.0, minimum_angle_penalty=0.85,
               angle_variance_penalty=(1 * D) ** 2)
    bt.grids[:] = 100
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)
    gpu, frac, _, _ = sweep_and_check(M, bt, se)
    assert frac == 65 / 81, frac
    ncell = abi.n_steps(se.offset_x, se.res_x) * abi.n_steps(se.offset_y, se.res_y)
    assert ncell > RED_MAX_TIES and (gpu[3] == 0).all() and (gpu[4] == ncell).all(), gpu[4]


def test_equal_probe_maxima_under_a_penalty_clamped_at_one(M):
    """every byte 100 and an angle penalty clamped at 1: every probed angle holds the same largest response, which is
    the best, tied at every angle of the centre cell; nothing is pruned"""
    bt = batch(1081, 3, 701, minimum_angle_penalty=1.0)
    bt.grids[:] = 100
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)
    gpu, frac, _, _ = sweep_and_check(M, bt, se)
    assert frac == 0.0
    assert (gpu[3] == 0).all() and (gpu[4] == 81).all(), gpu[4]


def test_responses_in_the_ambiguous_band(M):
    """6000 beams on grids of scattered 1s: a window sum of 1 is a response of 1 / 600 000 = 1.67e-6, inside the band
    near the 1e-6 DoubleEqual threshold in which the pre-filter always evaluates exactly.  In the odd matches the
    scan's cells at the centre candidate also hold 100, so that their best is high and angles are pruned."""
    bt = batch(6000, 4, 702)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    bt.grids[::2] = 0
    bt.grids[:] = np.maximum(bt.grids, np.random.default_rng(703).random(bt.grids.shape) < 2e-4)
    gpu, frac, sums, keep = sweep_and_check(M, bt, se)
    for b in range(0, bt.B, 2):
        assert (sums[b] == 1).any() and keep[b].all() and not keep[b + 1].all(), b


def test_cells_of_zero_sums_next_to_cells_that_are_not(M):
    """60 beams whose points lie far apart, the cells they hit from the centre candidate at the middle angle 100: the
    far angles are pruned, and many cells miss every one of those cells at every angle that is swept"""
    bt = batch(60, 8, 704)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    gpu, frac, sums, keep = sweep_and_check(M, bt, se)
    for b in range(bt.B):
        cell_max = sums[b][:, :, keep[b]].max(axis=2)
        assert not keep[b].all() and (cell_max == 0).any() and (cell_max > 0).any(), b
