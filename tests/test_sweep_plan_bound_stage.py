"""Where k_sweep_bound (csrc/karto_matcher.cu) reads the scan-local points and the summed-area table it places every
beam with: plan_sweep (csrc/karto_sweep_plan.cuh) stages them in shared memory after the pooled image when they fit
there (SweepPlan::bound_stage), and otherwise the bound reads them from global memory; either way the search is still
pruned.  Checked on the host, without a GPU (tests/sweep_plan_check.cu)."""
from test_sweep_plan import CFG2_SEARCH, D, OPTIN, WIN_STATIC, params, plan, plan_request  # noqa: F401 (plan: the driver)


def req(geom, search, n=1081, batch=1024, force=0, sat_valid=1):
    return plan_request(params(*geom), n, batch, search, force=force, sat_valid=sat_valid)


CFG2 = (1.5, 0.05, 0.03, 9.25)
LIMIT = OPTIN - WIN_STATIC - 512  # what the bound's dynamic shared memory may use


def angles(na, res=0.25 * D):
    return (0.75, 0.75, 0.05, 0.05, 0.5 * (na - 1) * res, res, 0)


def test_cfg2_stages_points_and_sat(plan):
    """cfg 2: 167 KB pooled image + 17 KB of points + 21 KB of SAT fit in the 227 KB"""
    (r,) = plan([req(CFG2, CFG2_SEARCH)])
    assert r["prune"] and r["skip_empty"] and r["bound_stage"]
    assert r["bound_smem"] == r["pool"]["bytes"] + 2 * 128 + 1081 * 16 + r["sat_bytes"]
    assert r["bound_smem"] <= LIMIT


def test_without_sat_only_points_are_staged(plan):
    """no valid SAT (no empty-window dropping): only the points go after the pooled image"""
    (r,) = plan([req(CFG2, CFG2_SEARCH, sat_valid=0)])
    assert r["prune"] and not r["skip_empty"] and r["bound_stage"]
    assert r["bound_smem"] == r["pool"]["bytes"] + 2 * 128 + 1081 * 16


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
        assert r["prune"] == r["pool"]["fits"], (t, r)
        staged = r["pool"]["bytes"] + 2 * 128 + 1081 * 16 + r["sat_bytes"] * r["skip_empty"]
        assert r["bound_stage"] == (r["prune"] and staged <= LIMIT), (t, r)
        assert r["bound_smem"] == (staged if r["bound_stage"] else r["pool"]["bytes"] + 2 * 128), (t, r)
        assert r["bound_smem"] <= LIMIT or not r["prune"], (t, r)
    kinds = [(r["prune"], r["bound_stage"]) for r in out]
    assert (1, 1) in kinds and (1, 0) in kinds and (0, 0) in kinds, kinds
    # ordered: staged, then pruned from global memory, then not pruned
    assert kinds == sorted(kinds, reverse=True), kinds


def test_dense_selector_does_not_stage(plan):
    """selector 3 sweeps every beam and every angle: no bound pass"""
    (r,) = plan([req(CFG2, CFG2_SEARCH, force=3)])
    assert not r["prune"] and not r["bound_stage"]
