"""The beam ranges of the angle bound (k_sweep_bound, csrc/karto_sweep_plan.cuh bound_chunks / bound_range): a round
of few units cuts each unit's beams into ranges whose block sums meet in one shared-memory row per unit.  Every case is
swept pruned and dense (every beam, every angle): equal byte for byte, equal to the C restatement, last_pruned_frac()
equal to the numpy bound and selection rule, empty_window_frac equal to the numpy count.  The sizes of rounds (b) and
(c) of every match are those of the numpy restatement of the rounds (tests/test_prune_group_bound.py), so the cases
are known to reach the splits they are meant to reach.

The cases: rounds (b) of 0, 4, 8, 25 and 65 angles and rounds (c) of 0, 4, 8 and 12; beam counts of 1 (every range
but one empty), 33 and 4500 (a flush of the packed sums inside a range); walls at 1 degree steps (beams on the group
pass's per-member fallback); and the benchmark's shape at batches of 1, 131 and 1024."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_gpu_matcher_prune import pruned_and_dense
from test_gpu_matcher_prune_chunks import check
from test_gpu_matcher_prune_lists import cfg2_inputs, dropped_beams
from test_gpu_matcher_prune_planes import scan_cells
from test_gpu_matcher_prune_tail import batch
from test_prune_bound import INVALID, angle_bounds, batch_cases, responses, walls
from test_prune_group_bound import GROUP, PROBE, group_bounds

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def round_sizes(bt, se):
    """(angles of round (a), of round (b), of round (c)) of every regular match, by the numpy restatement"""
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    out = []
    for grid, g, lut, base00, sums, n, se_, params, ch in batch_cases(bt, se):
        drop, _ = dropped_beams(grid, g, lut, base00, nx, ny)
        ubr = angle_bounds(grid, g.width_step, np.where(drop, INVALID, lut), base00, n, se_, params, ch)
        gub = group_bounds(grid, g.width_step, lut, base00, n, se_, params, ch)
        resp = responses(sums, n, se_, params, ch)
        na, ng = len(ubr), len(gub)
        members = [list(range(h * GROUP, min(h * GROUP + GROUP, na))) for h in range(ng)]
        order = sorted(range(ng), key=lambda h: (-gub[h], h))
        ev_a, top = [], 0
        while len(ev_a) < min(PROBE, na):
            ev_a += members[order[top]]
            top += 1
        f16 = sorted((ubr[k] for k in ev_a), reverse=True)[min(PROBE, na) - 1]
        ev_b = [k for h in order[top:] if gub[h] >= f16 for k in members[h]]
        probe = sorted(ev_a + ev_b, key=lambda k: (-ubr[k], k))[:min(PROBE, na)]
        L = resp[:, :, probe].max()
        n_c = 0
        if L - 0.1 > 1e-6:
            done = set(ev_a + ev_b)
            n_c = sum(1 for k in range(na) if k not in done and gub[k // GROUP] >= L - 0.1 - 1e-9)
        out.append((len(ev_a), len(ev_b), n_c))
    return out


@pytest.mark.parametrize("width, want", [(1.0, [(16, 65, 0)] * 2), (5.0, [(16, 4, 0), (16, 0, 0)]),
                                         (8.0, [(16, 4, 4)] * 2)])
def test_round_sizes(M, width, want):
    """every byte 100 and an angle penalty that falls to its 0.85 floor `width` degrees off the centre"""
    bt = batch(1081, 2, 810 + int(10 * width), minimum_distance_penalty=1.0, minimum_angle_penalty=0.85,
               angle_variance_penalty=(width * D) ** 2)
    bt.grids[:] = 100
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D)
    assert round_sizes(bt, se) == want
    check(M, bt, se)


@pytest.mark.parametrize("n, want", [(1, [(16, 4, 12), (16, 0, 8), (16, 0, 12)]), (33, [(16, 25, 0)] * 3),
                                     (4500, [(16, 8, 4), (16, 8, 4), (16, 8, 8)])])
def test_beam_counts(M, n, want):
    """scattered cells plus the scan's cells at the centre, 1 degree steps"""
    bt = batch(n, 3, 800 + n)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    bt.grids[:] = np.maximum(bt.grids, (np.random.default_rng(900 + n).random(bt.grids.shape) < 0.02) * 60)
    assert round_sizes(bt, se) == want
    check(M, bt, se)


def test_walls_on_the_group_fallback(M):
    """walls along the grid's edges and across row ends at 1 degree steps, a round (b) of 25 angles"""
    bt, _ = kv.probe_batch((1.5, 0.05, 0.03, 9.25), 1, seed=720, B=6)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    scan_cells(bt, se)
    walls(bt, np.random.default_rng(701))
    assert round_sizes(bt, se) == [(16, 25, 0)] * 6
    check(M, bt, se)


@pytest.mark.parametrize("B", [1, 131, 1024])
def test_cfg2_batches(pkg, M, B):
    """the benchmark's shape: pruned == dense byte for byte"""
    A = cfg2_inputs(pkg, range(4_000_000, 4_000_000 + B))
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 1, 0)
    m = M.ScanMatcher(A[0], A[1], max_batch=B, max_base_scans=1)
    m.set_scans(A[2], A[3])
    m.add_scans(A[4], A[5])
    _, frac = pruned_and_dense(m, A[6], se)
    m.close()
    assert 0.6 <= frac < 1.0, frac
