"""The group pass of the correlative sweep's angle pruning on the device (k_grid_pool<7>, k_sweep_bound's three modes,
k_prune_select and the on-demand empty-window count in csrc/karto_matcher.cu).  Every case is swept pruned and dense
(every beam, every angle): the results are equal byte for byte, last_pruned_frac() equals the numpy restatement of
the per-angle bound and the selection rule.  empty_window_frac of a pruned sweep is counted when it is read (its value
against the restatement is checked in tests/test_gpu_matcher_prune_lists.py); here it is the same on every read of the
same sweep and NaN once the sweep's inputs were replaced.

The cases: the cfg-2 matches; angle counts that leave the last group with 1 or 3 angles; angle steps so coarse
that every beam's origins spread past 3 cells across a group (the per-member fallback) and so fine that a group's
four origins mostly coincide; and a read of the statistics after the inputs were replaced, which reports NaN."""
import math

import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_gpu_matcher_prune import pruned_and_dense
from test_gpu_matcher_prune_lists import cfg2_inputs
from test_gpu_matcher_prune_planes import restated_pruned, scan_cells
from test_prune_bound import walls

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def sweep_and_check(M, bt, se):
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    m.set_kernel(0)
    m.correlate_scan(bt.centers, se)
    empty = m.last_stats()["empty_window_frac"]  # counted on demand after the pruned sweep
    assert m.last_stats()["empty_window_frac"] == empty and 0.0 <= empty <= 1.0
    _, frac = pruned_and_dense(m, bt.centers, se)
    m.close()
    na = abi.n_steps(se.angle_offset, se.angle_res)
    pruned, _ = restated_pruned(bt, se)
    assert frac == pruned / (float(bt.B) * na), (frac, pruned)
    return frac


@pytest.mark.parametrize("angle_offset_deg, angle_res_deg", [(20, 1), (20.25, 0.75), (20.5, 0.5), (4.5, 0.1), (40, 2)])
def test_group_sizes_and_spreads(M, angle_offset_deg, angle_res_deg):
    """41, 55, 83, 91 and 41 angles (the last group holds 1, 3, 3, 3 and 1 of them); 2 degree steps put every beam
    far from the sensor on the per-member fallback, 0.1 degree steps keep almost every group on one corner"""
    bt, _ = kv.probe_batch((1.5, 0.05, 0.03, 9.25), 1, seed=700 + int(angle_res_deg * 100), B=12)
    se = kv.window_search(bt, angle_offset=angle_offset_deg * D, angle_res=angle_res_deg * D)
    scan_cells(bt, se)
    walls(bt, np.random.default_rng(701))
    assert sweep_and_check(M, bt, se) > 0.0


def test_cfg2_matches(M, pkg):
    params, laser, ranges, poses, bran, bpos, _ = cfg2_inputs(pkg, range(3_000_000, 3_000_008))
    m = M.ScanMatcher(params, laser, max_batch=len(ranges), max_base_scans=1)
    m.set_scans(ranges, poses)
    m.add_scans(bran, bpos)
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m.correlate_scan(poses, se)
    empty = m.last_stats()["empty_window_frac"]
    _, frac = pruned_and_dense(m, poses, se)
    assert frac > 0.5 and empty > 0.0
    m.correlate_scan(poses, se)
    assert m.last_stats()["empty_window_frac"] == empty
    # a pruned sweep, then new scans before the statistics are read: the inputs of that sweep are gone
    m.correlate_scan(poses, se)
    m.set_scans(ranges, poses)
    assert math.isnan(m.last_stats()["empty_window_frac"])
    m.close()
