"""Which CorrelateScan searches plan_sweep (csrc/karto_sweep_plan.cuh) prunes by angle: the automatic choice is made
there alone, on the host, so it is checked without a GPU.  Pruned: one stride-1 32 x 32 candidate tile on a grid that
fits shared memory, with PRUNE_MIN_ANGLES..PRUNE_MAX_ANGLES angles of a whole search.  Not pruned: banded grids, the
stride-2 coarse stage, the fine stage's 3 x 3 x 11, angle subsets of a split sweep, the generic kernel and selector 3.
tests/sweep_plan_check.cu runs the plan."""
import pytest

from test_sweep_plan import CFG2_SEARCH, D, OPTIN, WIN_STATIC, params, plan, plan_request  # noqa: F401 (plan: the driver)


def req(geom, search, n=1081, batch=1024, k_first=0, na_override=-1, force=0):
    return plan_request(params(*geom), n, batch, search, k_first=k_first, na_override=na_override, force=force)


CFG2 = (1.5, 0.05, 0.03, 9.25)


def angles(na, res=0.25 * D):
    return (0.75, 0.75, 0.05, 0.05, 0.5 * (na - 1) * res, res, 0)


def test_cfg2_prunes_on_the_window_kernel(plan):
    (r,) = plan([req(CFG2, CFG2_SEARCH)])
    assert r["status"] == 0 and r["use_window"] and r["nbands"] == 1 and r["na"] == 181
    assert r["prune"] and r["pool"]["fits"] and r["bound_smem"] + WIN_STATIC <= OPTIN


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
    assert not r["prune"] and not r["pool"]["fits"]
