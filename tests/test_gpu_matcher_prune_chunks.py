"""The beam ranges of a pruned window sweep (k_sweep_window<LISTED>, csrc/karto_sweep_plan.cuh listed_chunks): the
probe and kept lists of few angles are split into beam ranges whose partial sums meet in shared memory.  Every case is
swept pruned and dense (set_kernel(3): every beam, every angle, no lists): equal byte for byte, equal to the C
restatement, last_pruned_frac() equal to the numpy bound and selection rule and empty_window_frac equal to the numpy
count of empty windows.

The cases: beam counts from 1 (one range, the rest empty) to 4500 (more than WIN_FLUSH_BEAMS in one range), kept lists
from none to a band of angles, an irregular lattice and an out-of-range centre next to pruned
matches, and batches of 1, 131 and 1024."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_gpu_matcher_prune import assert_matches_restatement, pruned_and_dense
from test_gpu_matcher_prune_lists import cfg2_inputs, dropped_beams
from test_gpu_matcher_prune_planes import scan_cells
from test_gpu_matcher_prune_tail import batch, sweep_and_check
from test_prune_bound import batch_cases

pytestmark = pytest.mark.gpu
PROBE = 16


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def empty_frac_of(M, bt, se):
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    m.correlate_scan(bt.centers, se)
    got = m.last_stats()["empty_window_frac"]
    m.close()
    return got


def check(M, bt, se):
    """sweep_and_check plus the empty-window fraction; -> the kept-list length of every regular match"""
    _, _, _, keep = sweep_and_check(M, bt, se)
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    na = abi.n_steps(se.angle_offset, se.angle_res)
    empties = sum(int(dropped_beams(grid, g, lut, base00, nx, ny)[1].sum())
                  for grid, g, lut, base00, *_ in batch_cases(bt, se))
    assert empty_frac_of(M, bt, se) == empties / (float(bt.B) * na * bt.laser_s.n_readings)
    return [int(k.sum()) - PROBE if not k.all() else 0 for k in keep]


@pytest.mark.parametrize("n", [1, 3, 4, 5, 31, 33, 1081, 4500])
def test_beam_counts(M, n):
    """scattered cells plus the scan's cells at the centre: a high best, so that the far angles are pruned"""
    bt = batch(n, 3, 800 + n)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    bt.grids[:] = np.maximum(bt.grids, (np.random.default_rng(900 + n).random(bt.grids.shape) < 0.02) * 60)
    check(M, bt, se)


@pytest.mark.parametrize("width", [1.0, 1.5, 2.0, 3.0, 4.0, 5.0])
def test_kept_lists_of_few_angles(M, width):
    """every byte 100 and an angle penalty that falls to its 0.85 floor `width` degrees off the centre: the probe holds
    the best 16 angles and the kept list the angles of the band left over, none at 1 degree (every other angle is
    pruned), more as the band widens"""
    bt = batch(1081, 2, 810 + int(10 * width), minimum_distance_penalty=1.0, minimum_angle_penalty=0.85,
               angle_variance_penalty=(width * D) ** 2)
    bt.grids[:] = 100
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)
    kept = check(M, bt, se)
    if width == 1.0:
        assert kept == [0, 0], kept


def test_irregular_lattice_next_to_pruned_matches(M):
    """match 0 on an irregular lattice (the generic sweep) and match 1 out of range, in one batch with pruned ones:
    pruned == dense byte for byte, every match equal to the restatement"""
    bt, se0 = kv.irregular_batch(1, seed=840, B=6)
    se = abi.Search(se0.offset_x, se0.offset_y, se0.res_x, se0.res_y, 20 * D, 1 * D, 1, 0)
    bt.centers[0] = kv.rounding_tie_center(bt, 0, se)
    scan_cells(bt, se)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu, frac = pruned_and_dense(m, bt.centers, se)
    m.close()
    assert frac > 0.0
    for b in range(bt.B):
        rc, res, _ = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)


@pytest.mark.parametrize("B", [1, 131, 1024])
def test_cfg2_batches(pkg, M, B):
    """the benchmark's shape at 1, 131 and 1024 matches: pruned == dense byte for byte"""
    seeds = range(3_000_000, 3_000_000 + B)
    A = cfg2_inputs(pkg, seeds)
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m = M.ScanMatcher(A[0], A[1], max_batch=B, max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    _, frac = pruned_and_dense(m, A[6], se)
    m.close()
    assert 0.6 <= frac < 1.0, frac
