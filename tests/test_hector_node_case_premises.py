"""The recorded Hector node cases (tests/hector_node_cases.py) still hold what they are named for (CPU).

Each per-node case exists to reach one field of a node's laser or map settings that the default cases leave at one
value: a start off the centre, a resolution and a level count, update factors, a laser's beam layout, its message
range limits and the node's distance filters.  A case that lost its premise would go on passing while no longer
telling a wrong field from a right one, so the premises are checked here against a numpy projection of the ranges
(laser_geometry's rule: range < 30 m in double, range >= range_min in float) and the node's squared thresholds."""
import math

import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P

CASES = cases.cases()
f32 = np.float32
INGEST_ROUND = 576  # beams the device ingest converts per round


def _projected(c):
    """[S, n] float32 ranges, the mask projectLaser keeps, and every beam's squared distance x * x + y * y (float32)."""
    amin, inc, rmin, _ = c["geometry"]
    r = np.asarray(c["ranges"], np.float32)
    a = float(amin) + np.arange(r.shape[1], dtype=np.float64) * float(inc)
    with np.errstate(all="ignore"):
        keep = (r.astype(np.float64) < 30.0) & (r >= f32(rmin))
        x = (r.astype(np.float64) * np.cos(a)).astype(np.float32)
        y = (r.astype(np.float64) * np.sin(a)).astype(np.float32)
        d = x * x + y * y
    return r, keep, x, d


def _params(name):
    """InitParams' values of the case, the node's defaults for the rest."""
    p = cases.hector_node.node_params(CASES[name]["params"])
    return {f: getattr(p, f) for f, _ in cases.hector_node.HectorNodeParams._fields_}


def _band(name, lo, hi, projected=True):
    """Per scan: beams whose range lies in [lo, hi) (and that projectLaser keeps, with `projected`)."""
    r, keep, _, _ = _projected(CASES[name])
    inside = (r >= f32(lo)) & (r < f32(hi))
    return (inside & keep if projected else inside).sum(1)


def _sqr(metres):
    """InitParams' squared threshold: squared in double, then rounded to float."""
    return f32(float(metres) * float(metres))


def _filtered(name):
    """Per scan: the projected beams rosPointCloudToDataContainer keeps with an identity mount (no z window)."""
    p = _params(name)
    _, keep, x, d = _projected(CASES[name])
    sqr_min, sqr_max = _sqr(p["laser_min_dist"]), _sqr(p["laser_max_dist"])
    use = float(p["use_max_scan_range"])
    with np.errstate(all="ignore"):
        ok = keep & (d > sqr_min) & (d < sqr_max) & ~((x < 0) & (d < f32(0.5))) & ~(d.astype(np.float64) > use * use)
    return ok


@pytest.mark.parametrize("name", ["start_asym", "start_asym_2", "res_0.075_odd_size"])
def test_asymmetric_origin(name):
    p = _params(name)
    assert p["map_start_x"] != p["map_start_y"]
    info = P.map_info(f32(p["map_resolution"]), int(p["map_size"]), p["map_start_x"], p["map_start_y"])
    assert info["origin_x"] != info["origin_y"]
    # origin = -(size * resolution * start) - resolution / 2 on each axis
    ext = p["map_size"] * p["map_resolution"]
    for axis in "xy":
        want = -ext * p[f"map_start_{axis}"] - p["map_resolution"] / 2
        assert abs(info[f"origin_{axis}"] - want) < 1e-4, (name, axis)


def test_walks_leave_the_centre():
    """The asymmetric-start walks move far enough that a swapped start moves their points across many cells."""
    for name in ("start_asym", "start_asym_2"):
        port = P.HectorNodePort(_params(name), CASES[name]["geometry"], CASES[name]["mount"])
        out = port.process(CASES[name]["ranges"], CASES[name]["stamps"])
        port.close()
        assert np.abs(out["pose"][:, :2]).max() > 0.1, name
        assert out["map_updated"].sum() >= 3, name


@pytest.mark.parametrize("name,res,dims", [("res_0.1_levels_1", 0.1, [256]),
                                           ("res_0.025_levels_4", 0.025, [512, 256, 128, 64]),
                                           ("res_0.075_odd_size", 0.075, [515, 257, 128, 64])])
def test_level_dimensions(name, res, dims):
    p = _params(name)
    assert f32(p["map_resolution"]) == f32(res) and p["map_multi_res_levels"] == len(dims)
    port = P.HectorNodePort(p, CASES[name]["geometry"], CASES[name]["mount"])
    assert [port.proc.level(l)[0].shape for l in range(len(dims))] == [(d, d) for d in dims]
    port.close()


def test_update_factors_differ():
    p, d = _params("factors"), P.HectorNodePort.DEFAULTS
    assert p["update_factor_free"] != p["update_factor_occupied"]
    assert p["update_factor_free"] != d["update_factor_free"]
    assert p["update_factor_occupied"] != d["update_factor_occupied"]


def test_laser_layouts():
    amin, inc, _, _ = CASES["ring_360"]["geometry"]
    assert CASES["ring_360"]["ranges"].shape[1] == 360 and f32(amin) == f32(-math.pi)
    assert abs(float(inc) * 360 - 2 * math.pi) < 1e-5
    assert CASES["ring_pitched"]["geometry"] == CASES["ring_360"]["geometry"]
    assert CASES["ring_pitched"]["params"]["laser_z_min_value"] == -0.3  # the pitched z window
    assert CASES["clockwise"]["geometry"][1] < 0 and CASES["clockwise"]["geometry"][0] > 0
    for name in ("ring_360", "clockwise", "ring_pitched"):
        assert (_filtered(name).sum(1) > 100).all(), name


def test_dense_scans_take_several_ingest_rounds():
    assert CASES["dense_4096"]["ranges"].shape[1] == 4096  # the node's per-scan maximum
    kept = _filtered("dense_4096").sum(1)
    assert (kept > 4 * INGEST_ROUND).all(), kept  # five rounds or more on every scan


def test_every_band_is_reached():
    """Per scan, the beams in each band of the message range limits and the node's filters."""
    # range_min 0.05: kept readings in [0.05, 0.1), which a range_min of 0.1 would drop; [0.03, 0.05) dropped
    assert f32(CASES["fields_lo"]["geometry"][2]) == f32(0.05)
    assert (_band("fields_lo", 0.05, 0.1) >= 20).all()
    assert (_band("fields_lo", 0.03, 0.05, projected=False) >= 5).all() and not _band("fields_lo", 0.0, 0.05).any()
    ok = _filtered("fields_lo")
    r = CASES["fields_lo"]["ranges"]
    assert ((ok & (r < f32(0.1))).sum(1) >= 20).all()  # laser_min_dist 0.03 lets them through
    # laser_min_dist 0.5: readings in (range_min, 0.5) that the default 0.2 would keep in part
    assert (_band("min_dist_0.5", 0.2, 0.5) >= 20).all()
    assert not (_filtered("min_dist_0.5") & (CASES["min_dist_0.5"]["ranges"] < f32(0.5))).any()
    # range_max 10 in the message: readings in (10, 30), which the 30 m cutoff keeps and the filters pass
    assert f32(CASES["fields_hi"]["geometry"][3]) == f32(10.0)
    hi = _filtered("fields_hi") & (CASES["fields_hi"]["ranges"] > f32(10.0))
    assert (hi.sum(1) >= 50).all()
    # range_max 40: readings on both sides of 30 m; [30, 40) is dropped by the cutoff and would pass every filter
    r40 = CASES["fields_40"]["ranges"]
    assert (_band("fields_40", 20.0, 30.0) >= 20).all()
    assert (_band("fields_40", 30.0, 40.0, projected=False) >= 20).all() and not _band("fields_40", 30.0, 40.0).any()
    assert (r40 == f32(30.0)).any(1).all() and (r40 == np.nextafter(f32(30.0), f32(0))).any(1).all()
    _, _, _, d40 = _projected(CASES["fields_40"])
    far = (r40 >= f32(30.0)) & (r40 < f32(40.0))
    assert (d40[far] < _sqr(50.0)).all() and (d40[far].astype(np.float64) <= 50.0 ** 2).all()
    # laser_max_dist 8 below use_max_scan_range 12: readings in (8, 12) the distance filter drops
    _, keep8, _, d8 = _projected(CASES["max_dist_8"])
    assert ((keep8 & (d8 >= _sqr(8.0)) & (d8.astype(np.float64) <= 144.0)).sum(1) >= 50).all()
    assert not (_filtered("max_dist_8") & (d8 >= _sqr(8.0))).any()
    # use_max_scan_range 5 below laser_max_dist: readings past 5 m that only it drops
    _, keep5, _, d5 = _projected(CASES["use_range_5"])
    assert ((keep5 & (d5.astype(np.float64) > 25.0) & (d5 < _sqr(30.0))).sum(1) >= 50).all()


@pytest.mark.parametrize("name", ["fields_lo", "min_dist_0.5", "fields_hi", "fields_40", "max_dist_8", "use_range_5",
                                  "ring_360", "dense_4096"])
def test_numpy_count_equals_the_port(name):
    """The numpy filter above is the node's rule: its per-scan count equals the restatement's kept-beam count."""
    c = CASES[name]
    assert c["mount"] == cases.mount()
    port = P.HectorNodePort(_params(name), c["geometry"], c["mount"])
    out = port.process(c["ranges"], c["stamps"])
    port.close()
    assert np.array_equal(out["n_points"], _filtered(name).sum(1)), name
