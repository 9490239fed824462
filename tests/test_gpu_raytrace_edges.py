"""Device tests of the Karto occupancy grid (K2c, karto_occgrid.cu) and the GMapping hit/visit map (K2b,
gmapping_map.cu) against the brute-force ray tracer (raytrace_reference.py), bit for bit, on the crafted cases of
raytrace_cases.py: every short segment in one launch, all octants, midpoint ties, lengths around the 32-lane stride
and up to 4000 cells, rounding ties, every range-filter edge, grids smaller than their rays, odd beam counts and
widths, far offsets, crafted counters for the threshold, storage maps narrower, as wide as and one column wider than
the published map, out-of-map beams and growing scan buffers.  The restatement (oracle/port.py) is compared too
wherever it can express the case."""
import dataclasses

import numpy as np
import pytest

import raytrace_cases as rc
import raytrace_reference as rr
from oracle import port

pytestmark = pytest.mark.gpu

KARTO = rc.karto_cases()
GMAP = rc.gmap_cases()


@pytest.fixture(scope="module")
def O(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("occgrid")


@pytest.fixture(scope="module")
def GM(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("gmapping")


def karto_same(a, b):
    """dimensions, cell visits, counters and cells exactly; the offset, a point reading made with the device's cos / sin,
    to 1e-9 m (DESIGN.md §4)"""
    assert (a["width"], a["height"], a["width_step"]) == (b["width"], b["height"], b["width_step"])
    assert np.allclose(a["offset"], b["offset"], rtol=0, atol=1e-9) and a["cell_visits"] == b["cell_visits"]
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("name", list(KARTO))
def test_karto_grid_equals_brute_force(O, name):
    c = KARTO[name]
    g = O.OccupancyGrid(c.laser, c.ranges, c.poses, c.resolution, bbox=c.bbox)
    a = g.arrays()
    b = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution, bbox=c.bbox)
    karto_same(a, b)
    for k in ("passes", "hits", "cells"):  # padding columns of the 8-aligned rows stay zero
        assert not a[k][:, a["width"]:].any(), k
    assert np.array_equal(g.ros_map(), rr.karto_ros_map(b["cells"], b["width"], b["height"]))
    if c.bbox is None:
        karto_same(a, port.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution))
    g.close()


def test_karto_batched_build_equals_single_grid(O):
    """the cases with CreateFromScans' own box through the batched build, which takes one laser per build and float32
    readings: each case's readings rounded to float32 (its traced end points still off half cells), one build per laser
    holding each of its cases twice, so that on the 16384-beam laser a warp's stride crosses from one grid to the next.
    Every grid's info and payload equal the single-grid handle's and the brute force's on the same readings."""
    groups = {}
    for name, c in KARTO.items():
        if c.bbox is None:
            key = tuple(getattr(c.laser, f) for f, _ in c.laser._fields_ if f != "offset_pose") + tuple(c.laser.offset_pose)
            groups.setdefault(key, []).append(dataclasses.replace(c, ranges=c.ranges.astype(np.float32).astype(np.float64)))
    assert sum(map(len, groups.values())) == len([c for c in KARTO.values() if c.bbox is None]) and len(groups) > 1
    for cases in groups.values():
        for c in cases:
            assert rc.karto_end_margins(c) >= rc.HALF_CELL_MARGIN
        twice = cases + cases
        out = O.create_from_scans_batch(cases[0].laser, [c.ranges for c in twice], [c.poses for c in twice],
                                        [c.resolution for c in twice])
        for k, c in enumerate(cases):
            g = O.OccupancyGrid(c.laser, c.ranges, c.poses, c.resolution)
            a = g.arrays()
            b = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution)
            karto_same(a, b)
            want = rr.karto_ros_map(b["cells"], b["width"], b["height"])
            assert np.array_equal(g.ros_map(), want)
            for info, payload in (out[k], out[k + len(cases)]):
                assert (info["width"], info["height"], info["width_step"]) == (a["width"], a["height"], a["width_step"])
                assert np.array_equal(info["offset"], a["offset"]) and info["cell_visits"] == a["cell_visits"]
                assert np.array_equal(payload, want)
            g.close()


def test_karto_threshold_on_crafted_counters(O):
    """UpdateCell on set counters: pass 0..3, hit / pass exactly 0.1 and just above, counters near 2^32 - 1"""
    las = rc.laser(1)
    g = O.OccupancyGrid(las, np.array([[1.0]]), np.array([[0.5, 0.5, 0.0]]), 1.0, bbox=[0.0, 0.0, 8.0, 3.0])
    assert (g.info.width, g.info.height, g.info.data_size) == (8, 3, 24)
    pairs = rc.THRESHOLD_PAIRS + [(0, 0)] * (24 - len(rc.THRESHOLD_PAIRS))
    passes = np.array([p for p, _ in pairs], np.uint32).reshape(3, 8)
    hits = np.array([h for _, h in pairs], np.uint32).reshape(3, 8)
    g.set_counters(passes, hits)
    g.update()
    a = g.arrays()
    assert np.array_equal(a["passes"], passes) and np.array_equal(a["hits"], hits)
    want = np.array([rr.update_cell(p, h) for p, h in pairs], np.uint8).reshape(3, 8)
    assert np.array_equal(a["cells"], want)
    assert want.reshape(-1)[8] == rr.FREE and want.reshape(-1)[9] == rr.OCCUPIED  # 10/100 is not above 0.1; 11/100 is
    assert np.array_equal(g.ros_map(), rr.karto_ros_map(want, 8, 3))
    g.close()


def test_karto_refuses_a_grid_whose_padded_size_overflows(pkg, O):
    """width * height = 2 147 441 940 fits in int32, width_step * height = 46344 * 46340 does not"""
    M, abi = pkg.load("matcher"), pkg.abi
    las = rc.laser(1)
    for box in ([0.0, 0.0, 46341.0, 46340.0], [0.0, 0.0, 65536.0, 65536.0]):
        with pytest.raises(M.B2SError) as e:
            O.OccupancyGrid(las, np.zeros((0, 1)), np.zeros((0, 3)), 1.0, bbox=box)
        assert e.value.status == abi.B2S_ERR_TOO_LARGE


def gmap_compare(dev, brute, restated=None):
    n, v, ax, ay = dev.cells()
    bn, bv, bax, bay = brute.cells()
    assert np.array_equal(n, bn) and np.array_equal(v, bv)
    if restated is not None:
        rn, rv, _, _ = restated.cells()
        assert np.array_equal(n, rn) and np.array_equal(v, rv)
    # float hit sums: a single hit is exact; n hits (device order) agree with the float64 sum within n ulps
    nf = n.reshape(-1)
    one = nf == 1
    assert np.array_equal(ax.reshape(-1)[one], bax.reshape(-1)[one])
    assert np.array_equal(ay.reshape(-1)[one], bay.reshape(-1)[one])
    many = np.flatnonzero(nf > 1)
    for i in many:
        tol = nf[i] * np.spacing(np.float32(brute.abs64[i]))
        assert abs(float(ax.reshape(-1)[i]) - brute.acc64_x[i]) <= tol
        assert abs(float(ay.reshape(-1)[i]) - brute.acc64_y[i]) <= tol
    return len(many)


@pytest.mark.parametrize("name", list(GMAP))
def test_gmapping_map_equals_brute_force(GM, name):
    case = GMAP[name]
    dev = GM.GMap(*case.bounds)
    brute, restated = rr.GMapReference(*case.bounds), port.PortGMap(*case.bounds)
    assert (dev.size_x, dev.size_y) == (brute.size_x, brute.size_y)
    multi = 0
    for call in case.calls:
        kw = dict(laser_xy=call.laser_xy, max_range=call.max_range, max_urange=call.max_urange)
        dev.compute_map(call.ranges, call.angles, **kw)
        assert brute.compute_map(call.ranges, call.angles, **kw) == 0
        restated.compute_map(call.ranges, call.angles, **kw)
        multi = gmap_compare(dev, brute, restated)
    if name == "growth":
        assert multi >= 5  # the float accumulators were exercised with several hits per cell
    first, second = dev.ros_map(), dev.ros_map()
    assert np.array_equal(first, second)
    assert np.array_equal(first, brute.ros_map())
    assert np.array_equal(first, restated.ros_map())
    dev.close()


def test_gmapping_out_of_map_beam_changes_nothing(pkg, GM):
    M, abi = pkg.load("matcher"), pkg.abi
    b = (-8.0, -8.0, 8.0, 8.0, rc.RES)
    dev, brute = GM.GMap(*b), rr.GMapReference(*b)
    r, a = rc.random_beams(b, (0.0, 0.0), 500, seed=2)
    dev.compute_map(r, a, (0.0, 0.0))
    brute.compute_map(r, a, (0.0, 0.0))
    before = [x.copy() for x in dev.cells()]
    for rng, ang in (([1.0, 128 * rc.RES], [0.3, 0.0]), ([2.0, 128.6 * rc.RES], [1.0, np.pi / 2])):
        with pytest.raises(M.B2SError) as e:
            dev.compute_map(np.array(rng), np.array(ang), (0.0, 0.0))
        assert e.value.status == abi.B2S_ERR_OUT_OF_RANGE
        assert brute.compute_map(np.array(rng), np.array(ang), (0.0, 0.0)) == -1
        assert all(np.array_equal(x, y) for x, y in zip(before, dev.cells()))
    # beams ending on the last and the first in-map cell are accepted
    edge_r, edge_a = np.array([127 * rc.RES, 128 * rc.RES, 127 * rc.RES]), np.array([0.0, np.pi, np.pi / 2])
    dev.compute_map(edge_r, edge_a, (0.0, 0.0))
    assert brute.compute_map(edge_r, edge_a, (0.0, 0.0)) == 0
    n, v, _, _ = dev.cells()
    assert n[128, 255] >= 1 and n[128, 0] >= 1 and n[255, 128] >= 1
    gmap_compare(dev, brute)
    assert np.array_equal(dev.ros_map(), brute.ros_map())
    dev.close()
