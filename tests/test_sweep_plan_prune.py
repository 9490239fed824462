"""Which CorrelateScan searches plan_sweep (csrc/karto_sweep_plan.cuh) prunes by angle: the automatic choice is made
there alone, on the host, so it is checked without a GPU.  Pruned: one stride-1 32 x 32 candidate tile on a grid that
fits shared memory, with PRUNE_MIN_ANGLES..PRUNE_MAX_ANGLES angles of a whole search.  Not pruned: banded grids, the
stride-2 coarse stage, the fine stage's 3 x 3 x 11, angle subsets of a split sweep, the generic kernel and selector 3."""
import importlib
import json
import math
import subprocess

import pytest

D = math.pi / 180
OPTIN, SMS, WIN_STATIC = 232_448, 132, 3_200  # as tests/test_sweep_plan.py

DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <sstream>
#include "karto_sweep_plan.cuh"
using namespace b2s;
int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    b2s_matcher_params p = {};
    b2s_search s = {};
    int n, batch, k_first, na_override, force;
    in >> p.search_size >> p.resolution >> p.smear_deviation >> p.range_threshold >> n >> batch >> s.offset_x >>
        s.offset_y >> s.res_x >> s.res_y >> s.angle_offset >> s.angle_res >> s.fine >> k_first >> na_override >> force;
    const b2s_grid_info g = grid_layout(p);
    const SweepPlan pl = plan_sweep(p, g, s, n, batch, k_first, na_override, force, true, false, (g.width_step + 3) / 4,
                                    (g.height + 3) / 4, %d, %d, %d);
    printf("{\"status\": %%d, \"na\": %%d, \"use_window\": %%d, \"nbands\": %%d, \"stride\": %%d, \"prune\": %%d, "
           "\"bound_smem\": %%zu, \"pool_fits\": %%d}\n", (int)pl.status, pl.na, (int)pl.use_window, pl.nbands, pl.stride,
           (int)pl.prune, pl.bound_smem, (int)pool_fits(g, %d, %d));
  }
  return 0;
}
""" % (SMS, OPTIN, WIN_STATIC, OPTIN, WIN_STATIC)


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    d = tmp_path_factory.mktemp("prune_plan")
    src, exe = d / "prune_plan.cu", str(d / "prune_plan")
    src.write_text(DRIVER)
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", build.os.path.join(build.HERE, "csrc"), "-I", build.os.path.join(build.HERE, "..", "include"),
                           str(src), "-o", exe])

    def run(reqs):
        out = subprocess.run([exe], input="".join(r + "\n" for r in reqs), capture_output=True, text=True, check=True)
        return [json.loads(line) for line in out.stdout.splitlines()]

    return run


def req(geom, search, n=1081, batch=1024, k_first=0, na_override=-1, force=0):
    return " ".join(repr(v) for v in (*geom, n, batch, *search, k_first, na_override, force))


CFG2 = (1.5, 0.05, 0.03, 9.25)
CFG2_SEARCH = (0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 0)


def angles(na, res=0.25 * D):
    return (0.75, 0.75, 0.05, 0.05, 0.5 * (na - 1) * res, res, 0)


def test_cfg2_prunes_on_the_window_kernel(plan):
    (r,) = plan([req(CFG2, CFG2_SEARCH)])
    assert r["status"] == 0 and r["use_window"] and r["nbands"] == 1 and r["na"] == 181
    assert r["prune"] and r["pool_fits"] and r["bound_smem"] + WIN_STATIC <= OPTIN


def test_selectors(plan):
    """0 picks (pruned), 1 generic, 2 window (pruned), 3 every beam and every angle"""
    out = plan([req(CFG2, CFG2_SEARCH, force=k) for k in range(4)])
    assert [r["prune"] for r in out] == [1, 0, 1, 0]


def test_angle_counts(plan):
    out = plan([req(CFG2, angles(na)) for na in (31, 33, 1023, 1025)] +
               [req(CFG2, angles(32, 1 * D)), req(CFG2, angles(1024, 0.01 * D))])
    assert [r["na"] for r in out] == [31, 33, 1023, 1025, 32, 1024]
    assert [r["prune"] for r in out] == [0, 1, 1, 0, 1, 1]


def test_stages_and_subsets_that_do_not_prune(plan):
    r = 1.0 / (1.0 / 0.05)
    coarse = (0.5 * 30 * r, 0.5 * 30 * r, 2 * r, 2 * r, 20 * D, 2 * D, 0)  # MatchScan's coarse stage: stride 2
    fine = (r, r, r, r, 1 * D, 0.2 * D, 1)  # its fine stage: 3 x 3 x 11
    out = plan([req(CFG2, coarse), req(CFG2, fine),
                req(CFG2, CFG2_SEARCH, k_first=0, na_override=181),  # the whole range as a split sweep's subset
                req(CFG2, CFG2_SEARCH, k_first=90, na_override=91),
                req(CFG2, (1.0, 1.0, 0.05, 0.05, 22.5 * D, 0.25 * D, 0))])  # 41 x 41 candidates: two tiles
    assert all(o["status"] == 0 and o["use_window"] for o in out), out
    assert out[0]["stride"] == 2 and out[1]["na"] == 11
    assert [o["prune"] for o in out] == [0, 0, 0, 0, 0]


@pytest.mark.parametrize("geom", [(1.5, 0.025, 0.03, 9.25), (1.5, 0.05, 0.03, 12.0)])
def test_banded_grids_do_not_prune(plan, geom):
    """cfg 4's 0.025 m grid and a 12 m range threshold: grids swept in row bands, pooled image too large"""
    (r,) = plan([req(geom, (0.75, 0.75, geom[1], geom[1], 22.5 * D, 0.25 * D, 0))])
    assert r["status"] == 0 and r["use_window"] and r["nbands"] > 1
    assert not r["prune"] and not r["pool_fits"]
