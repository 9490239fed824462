"""Where k_sweep_bound (csrc/karto_matcher.cu) reads the scan-local points and the summed-area table it places every
beam with: plan_sweep (csrc/karto_sweep_plan.cuh) stages them in shared memory after the pooled image when they fit
there (SweepPlan::bound_stage), and otherwise the bound reads them from global memory; either way the search is still
pruned.  Checked on the host, without a GPU."""
import importlib
import json
import math
import subprocess

import pytest

D = math.pi / 180
OPTIN, SMS, WIN_STATIC = 232_448, 132, 3_200  # H100 opt-in shared memory per block, SMs, k_sweep_window's static

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
    int n, batch, force, sat_valid;
    in >> p.search_size >> p.resolution >> p.smear_deviation >> p.range_threshold >> n >> batch >> s.offset_x >>
        s.offset_y >> s.res_x >> s.res_y >> s.angle_offset >> s.angle_res >> s.fine >> force >> sat_valid;
    const b2s_grid_info g = grid_layout(p);
    const int sbx = (g.width_step + 3) / 4, sby = (g.height + 3) / 4;
    const SweepPlan pl = plan_sweep(p, g, s, n, batch, 0, -1, force, sat_valid != 0, false, sbx, sby, %d, %d, %d);
    printf("{\"status\": %%d, \"na\": %%d, \"prune\": %%d, \"skip_empty\": %%d, \"bound_stage\": %%d, "
           "\"bound_smem\": %%zu, \"pool_fits\": %%d, \"pool_bytes\": %%d, \"sat_bytes\": %%zu}\n", (int)pl.status, pl.na,
           (int)pl.prune, (int)pl.skip_empty, (int)pl.bound_stage, pl.bound_smem, (int)pool_fits(g, %d, %d),
           pool_bytes(g), sizeof(uint16_t) * sat_stride(sbx, sby));
  }
  return 0;
}
""" % (SMS, OPTIN, WIN_STATIC, OPTIN, WIN_STATIC)


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    d = tmp_path_factory.mktemp("bound_stage_plan")
    src, exe = d / "bound_stage_plan.cu", str(d / "bound_stage_plan")
    src.write_text(DRIVER)
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", build.os.path.join(build.HERE, "csrc"), "-I", build.os.path.join(build.HERE, "..", "include"),
                           str(src), "-o", exe])

    def run(reqs):
        out = subprocess.run([exe], input="".join(r + "\n" for r in reqs), capture_output=True, text=True, check=True)
        return [json.loads(line) for line in out.stdout.splitlines()]

    return run


def req(geom, search, n=1081, batch=1024, force=0, sat_valid=1):
    return " ".join(repr(v) for v in (*geom, n, batch, *search, force, sat_valid))


CFG2 = (1.5, 0.05, 0.03, 9.25)
CFG2_SEARCH = (0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 0)
LIMIT = OPTIN - WIN_STATIC - 512  # what the bound's dynamic shared memory may use


def angles(na, res=0.25 * D):
    return (0.75, 0.75, 0.05, 0.05, 0.5 * (na - 1) * res, res, 0)


def test_cfg2_stages_points_and_sat(plan):
    """cfg 2: 167 KB pooled image + 17 KB of points + 21 KB of SAT fit in the 227 KB"""
    (r,) = plan([req(CFG2, CFG2_SEARCH)])
    assert r["prune"] and r["skip_empty"] and r["bound_stage"]
    assert r["bound_smem"] == r["pool_bytes"] + 2 * 128 + 1081 * 16 + r["sat_bytes"]
    assert r["bound_smem"] <= LIMIT


def test_without_sat_only_points_are_staged(plan):
    """no valid SAT (no empty-window dropping): only the points go after the pooled image"""
    (r,) = plan([req(CFG2, CFG2_SEARCH, sat_valid=0)])
    assert r["prune"] and not r["skip_empty"] and r["bound_stage"]
    assert r["bound_smem"] == r["pool_bytes"] + 2 * 128 + 1081 * 16


def test_shapes_that_pruned_still_prune(plan):
    """33 and 1023 angles, 1024 angles at 0.01 deg, and cfg 2: pruned, points and SAT staged"""
    out = plan([req(CFG2, angles(na)) for na in (33, 1023)] + [req(CFG2, angles(1024, 0.01 * D)), req(CFG2, CFG2_SEARCH)])
    assert [r["na"] for r in out] == [33, 1023, 1024, 181]
    assert all(r["status"] == 0 and r["prune"] and r["bound_stage"] for r in out), out


def test_range_thresholds_near_the_pool_limit(plan):
    """Growing the range threshold grows the grid: first the points and SAT stop fitting beside the pooled image (the
    bound reads them from global memory and the search is still pruned), then the pooled image itself stops fitting
    (no pruning).  Every threshold whose pooled image fits is pruned, staged or not."""
    thresholds = [9.25 + 0.05 * i for i in range(0, 60)]
    out = plan([req((1.5, 0.05, 0.03, t), CFG2_SEARCH) for t in thresholds])
    for t, r in zip(thresholds, out):
        assert r["status"] == 0, (t, r)
        assert r["prune"] == r["pool_fits"], (t, r)
        staged = r["pool_bytes"] + 2 * 128 + 1081 * 16 + r["sat_bytes"] * r["skip_empty"]
        assert r["bound_stage"] == (r["prune"] and staged <= LIMIT), (t, r)
        assert r["bound_smem"] == (staged if r["bound_stage"] else r["pool_bytes"] + 2 * 128), (t, r)
        assert r["bound_smem"] <= LIMIT or not r["prune"], (t, r)
    kinds = [(r["prune"], r["bound_stage"]) for r in out]
    assert (1, 1) in kinds and (1, 0) in kinds and (0, 0) in kinds, kinds
    # ordered: staged, then pruned from global memory, then not pruned
    assert kinds == sorted(kinds, reverse=True), kinds


def test_dense_selector_does_not_stage(plan):
    """selector 3 sweeps every beam and every angle: no bound pass"""
    (r,) = plan([req(CFG2, CFG2_SEARCH, force=3)])
    assert not r["prune"] and not r["bound_stage"]
