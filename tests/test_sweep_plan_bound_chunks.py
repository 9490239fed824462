"""The work items of the angle bound (csrc/karto_sweep_plan.cuh: split_chunks<32, 128>, split_range<32>,
SweepPlan::bound_rows / group_rows): a round of few units cuts each unit's beams into ranges on multiples of 32, whose
block sums k_sweep_bound adds into one shared-memory row per unit.  Checked on the host, without a GPU
(tests/sweep_plan_check.cu): the ranges tile 0..n without overlap, a round gets about two items per warp with at least
BOUND_CHUNK_MIN_BEAMS beams per range on average, a round of more units than rows is one item per unit, and the rows
fit beside the staged data at the benchmark's shape."""
import numpy as np
import pytest

from test_sweep_plan import CFG2, CFG2_SEARCH, plan, plan_request  # noqa: F401 (plan: the driver fixture)

WARPS = 16  # WIN_THREADS / 32
MIN_BEAMS = 128  # BOUND_CHUNK_MIN_BEAMS
LIMIT = 232448 - 3200 - 512  # the H100's opt-in shared memory less the window kernel's static arrays and slack


def check_tiling(n, C, ranges):
    assert len(ranges) == C
    seen = np.zeros(n, dtype=np.int64)
    prev = 0
    for lo, hi in ranges:
        assert lo == prev and lo % 32 == 0 and lo <= hi <= n, (n, C, ranges)
        assert hi % 32 == 0 or hi == n, (n, C, ranges)
        seen[lo:hi] += 1
        prev = hi
    assert prev == n and (seen == 1).all(), (n, C, ranges)


def test_ranges_tile_the_beams(plan):
    cases = [(n, C) for n in (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1081, 2048, 2049, 4500, 9000)
             for C in range(1, 17)]
    for (n, C), r in zip(cases, plan([f"ranges 32 {n} {C}" for n, C in cases])):
        check_tiling(n, C, r["ranges"])


def test_chunk_counts(plan):
    """about two items per warp for every unit count from 1 to the 46 groups of the benchmark, within the rows"""
    reqs, want = [], []
    for n in (1, 31, 32, 33, 255, 256, 1081, 4500):
        for units in range(0, 47):
            for rows in (0, 1, 16, 31):
                reqs.append(f"chunks 32 {units} {n} {WARPS} {rows}")
                want.append((units, n, rows))
    for (units, n, rows), r in zip(want, plan(reqs)):
        C = r["chunks"]
        assert C >= 1
        if units == 0 or units > rows or n < 2 * MIN_BEAMS:  # no rows for the round, or too few beams for two ranges
            assert C == 1, (units, n, rows, C)
            continue
        assert units * C >= 2 * WARPS or C == n // MIN_BEAMS, (units, n, rows, C)  # about two items per warp
        assert units * (C - 1) < 2 * WARPS, (units, n, rows, C)                  # and no more ranges than that needs
        assert n // C >= MIN_BEAMS, (units, n, rows, C)                           # enough beams per range
    got = plan([f"chunks 32 {u} {n} {WARPS} 31" for u, n in ((1, 1), (1, 31), (1, 32), (1, 33), (16, 1081), (8, 1081),
                                                        (12, 1081), (20, 1081), (4, 1081), (46, 1081), (1, 4500),
                                                        (16, 4500), (31, 1081), (32, 1081))])
    assert [r["chunks"] for r in got] == [1, 1, 1, 1, 2, 4, 3, 2, 8, 1, 32, 2, 2, 1]


def test_cfg2_rows_fit_beside_the_staged_data(plan):
    """at the benchmark's shape the bound stages 201 KB (pooled image, points, summed-area table) and still holds
    31 rows; the group pass (7x7 image and points) too"""
    (pl,) = plan([plan_request(CFG2, 1081, 1024, CFG2_SEARCH)])
    assert pl["prune"] and pl["group"] and pl["bound_stage"] and pl["group_stage"] and pl["skip_empty"], pl
    assert pl["bound_rows"] == 31 and pl["group_rows"] == 31, pl
    assert pl["bound_smem"] + 31 * 256 == pl["pool"]["bytes"] + 256 + pl["stage"] + 31 * 256 <= LIMIT, pl
    assert pl["group_smem"] + 31 * 256 == pl["pool7"]["bytes"] + 256 + pl["stage7"] + 31 * 256 <= LIMIT, pl


@pytest.mark.parametrize("n", [1081, 2000, 2400, 2600])
def test_rows_fall_back_when_they_do_not_fit(plan, n):
    """more beams stage more points: the rows that fit shrink to none, and a round of more units than rows is one item
    per unit (bound_chunks); the bound never asks for more shared memory than there is"""
    (pl,) = plan([plan_request(CFG2, n, 1024, CFG2_SEARCH)])
    assert pl["prune"], pl
    for smem, rows, base in ((pl["bound_smem"], pl["bound_rows"], pl["pool"]["bytes"] + 256 + (pl["stage"] if pl["bound_stage"] else 0)),
                             (pl["group_smem"], pl["group_rows"], pl["pool7"]["bytes"] + 256 + (pl["stage7"] if pl["group_stage"] else 0))):
        assert 0 <= rows <= 31 and smem == base and smem + 256 * rows <= LIMIT, pl
        assert rows == 31 or base + 256 * (rows + 1) > LIMIT, pl
    (c,) = plan([f"chunks 32 {pl['bound_rows'] + 1} {n} {WARPS} {pl['bound_rows']}"])
    assert c["chunks"] == 1
    if n == 2400:
        assert pl["bound_stage"] and pl["bound_rows"] < 16, pl  # the probe round of 16 angles is one item per angle
