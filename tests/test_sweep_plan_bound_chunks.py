"""The work items of the angle bound (csrc/karto_sweep_plan.cuh: bound_chunks, bound_range, SweepPlan::bound_rows /
group_rows): a round of few units cuts each unit's beams into ranges on multiples of 32, whose block sums k_sweep_bound
adds into one shared-memory row per unit.  Checked on the host, without a GPU: the ranges tile 0..n without overlap,
a round gets about two items per warp with at least BOUND_CHUNK_MIN_BEAMS beams per range on average, a round of more
units than rows is one item per unit, and the rows fit beside the staged data at the benchmark's shape."""
import importlib
import json
import subprocess

import numpy as np
import pytest

WARPS = 16  # WIN_THREADS / 32
MIN_BEAMS = 128  # BOUND_CHUNK_MIN_BEAMS
LIMIT = 232448 - 3200 - 512  # the H100's opt-in shared memory less the window kernel's static arrays and slack

DRIVER = r"""
#include <cmath>
#include <cstdio>
#include <iostream>
#include <sstream>
#include "karto_sweep_plan.cuh"
using namespace b2s;
// request: plan <n> <smem_optin>                  -> the benchmark search's bound budget at n beams
//          chunks <units> <n> <warps> <rows>      -> {"chunks": C}
//          ranges <n> <C>                         -> {"ranges": [[lo, hi], ...]}
int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    in >> cmd;
    if (cmd == "plan") {  // the benchmark's search: 31 x 31 x 181 on a 0.05 m grid
      int n, optin;
      in >> n >> optin;
      b2s_matcher_params p = {};
      p.search_size = 1.5; p.resolution = 0.05; p.smear_deviation = 0.03; p.range_threshold = 9.25;
      b2s_search s = {};
      s.offset_x = s.offset_y = 0.75; s.res_x = s.res_y = 0.05; s.angle_offset = 22.5 * M_PI / 180; s.angle_res = 0.25 * M_PI / 180;
      const b2s_grid_info g = grid_layout(p);
      const SweepPlan pl = plan_sweep(p, g, s, n, 1024, 0, -1, 0, true, false, (g.width_step + 3) / 4,
                                      (g.height + 3) / 4, 132, optin, 3200);
      printf("{\"prune\": %d, \"group\": %d, \"bound_stage\": %d, \"group_stage\": %d, \"skip_empty\": %d, "
             "\"bound_rows\": %d, \"group_rows\": %d, \"bound_smem\": %zu, \"group_smem\": %zu, \"pool\": %d, "
             "\"pool7\": %d, \"stage\": %zu, \"stage7\": %zu}\n",
             (int)pl.prune, (int)pl.group, (int)pl.bound_stage, (int)pl.group_stage, (int)pl.skip_empty,
             pl.bound_rows, pl.group_rows, pl.bound_smem, pl.group_smem, pool_bytes(g), pool7_bytes(g),
             bound_stage_bytes(n, pl.skip_empty, (g.width_step + 3) / 4, (g.height + 3) / 4),
             bound_stage_bytes(n, false, 0, 0));
    } else if (cmd == "chunks") {
      int units, n, warps, rows;
      in >> units >> n >> warps >> rows;
      printf("{\"chunks\": %d}\n", bound_chunks(units, n, warps, rows));
    } else {
      int n, C;
      in >> n >> C;
      printf("{\"ranges\": [");
      for (int c = 0; c < C; c++) {
        int lo, hi;
        bound_range(n, c, C, lo, hi);
        printf("%s[%d, %d]", c ? ", " : "", lo, hi);
      }
      printf("]}\n");
    }
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    d = tmp_path_factory.mktemp("bound_chunks")
    src, exe = d / "bound_chunks.cu", str(d / "bound_chunks")
    src.write_text(DRIVER)
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", build.os.path.join(build.HERE, "csrc"), "-I", build.os.path.join(build.HERE, "..", "include"),
                           str(src), "-o", exe])

    def go(reqs):
        out = subprocess.run([exe], input="".join(r + "\n" for r in reqs), capture_output=True, text=True, check=True)
        return [json.loads(line) for line in out.stdout.splitlines()]

    return go


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


def test_ranges_tile_the_beams(run):
    cases = [(n, C) for n in (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1081, 2048, 2049, 4500, 9000)
             for C in range(1, 17)]
    for (n, C), r in zip(cases, run([f"ranges {n} {C}" for n, C in cases])):
        check_tiling(n, C, r["ranges"])


def test_chunk_counts(run):
    """about two items per warp for every unit count from 1 to the 46 groups of the benchmark, within the rows"""
    reqs, want = [], []
    for n in (1, 31, 32, 33, 255, 256, 1081, 4500):
        for units in range(0, 47):
            for rows in (0, 1, 16, 31):
                reqs.append(f"chunks {units} {n} {WARPS} {rows}")
                want.append((units, n, rows))
    for (units, n, rows), r in zip(want, run(reqs)):
        C = r["chunks"]
        assert C >= 1
        if units == 0 or units > rows or n < 2 * MIN_BEAMS:  # no rows for the round, or too few beams for two ranges
            assert C == 1, (units, n, rows, C)
            continue
        assert units * C >= 2 * WARPS or C == n // MIN_BEAMS, (units, n, rows, C)  # about two items per warp
        assert units * (C - 1) < 2 * WARPS, (units, n, rows, C)                  # and no more ranges than that needs
        assert n // C >= MIN_BEAMS, (units, n, rows, C)                           # enough beams per range
    got = run([f"chunks {u} {n} {WARPS} 31" for u, n in ((1, 1), (1, 31), (1, 32), (1, 33), (16, 1081), (8, 1081),
                                                        (12, 1081), (20, 1081), (4, 1081), (46, 1081), (1, 4500),
                                                        (16, 4500), (31, 1081), (32, 1081))])
    assert [r["chunks"] for r in got] == [1, 1, 1, 1, 2, 4, 3, 2, 8, 1, 32, 2, 2, 1]


def test_cfg2_rows_fit_beside_the_staged_data(run):
    """at the benchmark's shape the bound stages 201 KB (pooled image, points, summed-area table) and still holds
    31 rows; the group pass (7x7 image and points) too"""
    (pl,) = run(["plan 1081 232448"])
    assert pl["prune"] and pl["group"] and pl["bound_stage"] and pl["group_stage"] and pl["skip_empty"], pl
    assert pl["bound_rows"] == 31 and pl["group_rows"] == 31, pl
    assert pl["bound_smem"] + 31 * 256 == pl["pool"] + 256 + pl["stage"] + 31 * 256 <= LIMIT, pl
    assert pl["group_smem"] + 31 * 256 == pl["pool7"] + 256 + pl["stage7"] + 31 * 256 <= LIMIT, pl


@pytest.mark.parametrize("n", [1081, 2000, 2400, 2600])
def test_rows_fall_back_when_they_do_not_fit(run, n):
    """more beams stage more points: the rows that fit shrink to none, and a round of more units than rows is one item
    per unit (bound_chunks); the bound never asks for more shared memory than there is"""
    (pl,) = run([f"plan {n} 232448"])
    assert pl["prune"], pl
    for smem, rows, base in ((pl["bound_smem"], pl["bound_rows"], pl["pool"] + 256 + (pl["stage"] if pl["bound_stage"] else 0)),
                             (pl["group_smem"], pl["group_rows"], pl["pool7"] + 256 + (pl["stage7"] if pl["group_stage"] else 0))):
        assert 0 <= rows <= 31 and smem == base and smem + 256 * rows <= LIMIT, pl
        assert rows == 31 or base + 256 * (rows + 1) > LIMIT, pl
    (c,) = run([f"chunks {pl['bound_rows'] + 1} {n} {WARPS} {pl['bound_rows']}"])
    assert c["chunks"] == 1
    if n == 2400:
        assert pl["bound_stage"] and pl["bound_rows"] < 16, pl  # the probe round of 16 angles is one item per angle
