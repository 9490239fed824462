"""The angle-pruning bound over the residue-split pooled image (k_grid_pool's four planes, k_sweep_bound's packed
corner sums in csrc/karto_matcher.cu) on the device.  Every case is swept pruned and dense (every beam, every angle):
the results are equal byte for byte, and last_pruned_frac() equals the numpy restatement of the bound and the
selection rule (tests/test_prune_bound.py) over the beams the lists keep.

The cases: grids of every width_step class the bound's plane rows can have (width_step % 32 = 0, 8, 16, 24; width_step
/ 4 is even, so its residue modulo 4 is 0 or 2), with windows that leave the grid on every side and isolated cells at
window corners and block edges; window origins of every plane and word alignment (origin modulo 16); a small grid
whose interior windows reach both ends of the data; and grids of 127 in every byte with 4500 beams, the largest pooled
value on every corner of every beam, past the bound's packed-u16 flush."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_gpu_matcher_prune import pruned_and_dense
from test_gpu_matcher_prune_lists import dropped_beams
from test_prune_bound import INVALID, angle_bounds, batch_cases, kept_angles, responses, walls

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def restated_pruned(bt, se):
    """angles left out over the whole batch by the numpy bound and k_prune_probe / k_prune_select's rule; the matches
    the pruned sweep does not take (no result, or an irregular lattice) leave out none"""
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    pruned, origins = 0, []
    for grid, g, lut, base00, sums, n, se_, params, ch in batch_cases(bt, se):
        drop, _ = dropped_beams(grid, g, lut, base00, nx, ny)
        ubr = angle_bounds(grid, g.width_step, np.where(drop, INVALID, lut), base00, n, se_, params, ch)
        pruned += int((~kept_angles(ubr, responses(sums, n, se_, params, ch))).sum())
        a = ((base00 + lut.astype(np.int64) + 2**31) % 2**32) - 2**31
        origins.append(a[~drop])
    return pruned, np.concatenate(origins) if origins else np.zeros(0, dtype=np.int64)


def scan_cells(bt, se):
    """100 at the cells the scan hits from the centre candidate at the middle angle, inside the grid: a best response
    well above 0.1, so that angles far from it are left out, on top of whatever the grid holds"""
    ws, na = bt.g.width_step, abi.n_steps(se.angle_offset, se.angle_res)
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    for b in range(bt.B):
        gx, gy = bt.cells(b, se)
        lut = bt.lut(b, se)[na // 2]
        f = int(gx[0, 0] + gy[0, 0] * ws) + (ny // 2) * ws + nx // 2 + lut[lut != INVALID].astype(np.int64)
        bt.grids[b][f[(f >= 0) & (f < bt.g.data_size)]] = 100


def sweep_and_check(M, bt, se):
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    _, frac = pruned_and_dense(m, bt.centers, se)
    m.close()
    na = abi.n_steps(se.angle_offset, se.angle_res)
    pruned, origins = restated_pruned(bt, se)
    assert frac == pruned / (float(bt.B) * na), (frac, pruned)
    return frac, origins


def interior(a, g):
    """the windows k_sweep_bound sums without the range test (win_origin_class: within 112 bytes of the grid)"""
    span = 31 * g.width_step + 32 + 8
    return (a - 8 >= -112) & (a + span <= g.data_size + 112)


@pytest.mark.parametrize("rt", [8.6, 8.8, 8.95, 9.25])
def test_width_step_classes(M, rt):
    """width_step 384, 392, 400 and 408 (the benchmark's): walls along every grid edge and across row ends, isolated
    cells at window corners; windows of every plane and word alignment among the interior ones"""
    bt, _ = kv.probe_batch((1.5, 0.05, 0.03, rt), 1, seed=600 + int(rt * 100), B=16)
    assert bt.g.width_step % 32 == {8.6: 0, 8.8: 8, 8.95: 16, 9.25: 24}[rt]
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    walls(bt, np.random.default_rng(601))
    frac, a = sweep_and_check(M, bt, se)
    assert frac > 0.0
    inner = a[interior(a, bt.g)]
    assert set(np.unique(inner % 16)) == set(range(16))
    assert (~interior(a, bt.g)).any()  # and edge windows, read with the range test


def test_small_grid_windows_near_both_ends(M):
    """a 0.3 m range threshold (width_step 48, 47 rows): windows of 32 rows, readings that leave the grid on every
    side, and interior windows that start above the grid or end within a few bytes of its last byte"""
    bt, _ = kv.probe_batch((1.5, 0.05, 0.03, 0.3), 1, seed=610, B=16)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    walls(bt, np.random.default_rng(611))
    frac, a = sweep_and_check(M, bt, se)
    assert frac > 0.0
    g = bt.g
    inner = a[interior(a, g)]
    assert inner.size and inner.min() < 0 and inner.max() + 31 * g.width_step + 31 >= g.data_size


def test_largest_pooled_value_past_the_flush(M):
    """127 in every byte and 4500 beams: every corner sum adds 127 per beam, each u16 lane of the packed sums takes
    1016 per 32 beams placed, and an angle flushes them twice before its end"""
    bt, _ = kv.uniform_batch(4500, 127, B=2)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)
    frac, a = sweep_and_check(M, bt, se)
    assert frac > 0.0 and interior(a, bt.g).all()  # only the angle penalty separates the angles
