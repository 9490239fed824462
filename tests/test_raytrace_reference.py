"""CPU tests pinning the brute-force ray tracer (raytrace_reference.py) to the C restatement (oracle/port.py) and, where
oracle/_ref is built, to the reference's own TraceLine and gridLine: segment by segment, then on every crafted case of
raytrace_cases.py that the restatement can express (counters, cells, cell visits and published maps).  The device
tests (test_gpu_raytrace_edges.py) then compare the kernels against the same brute force."""
import math

import numpy as np
import pytest

import raytrace_cases as rc
import raytrace_reference as rr
from oracle import port, ref, ref_gmapping

SEGMENTS = [(dx, dy) for dx in range(-40, 41) for dy in range(-40, 41)]
LONG_SEGMENTS = [(1000, 37), (-1000, 999), (4000, -129), (129, 4000), (-3, -4000), (4000, 4000), (65, 64), (-97, 32),
                 (20000, 7), (-12345, 6789)]


def test_karto_trace_line_equals_restatement():
    for x0, y0 in ((0, 0), (3, -2)):
        for dx, dy in SEGMENTS + LONG_SEGMENTS:
            want = port.trace_line(1 << 20, 1 << 20, x0 + 50000, y0 + 50000, x0 + 50000 + dx, y0 + 50000 + dy)
            got = rr.trace_line(x0, y0, x0 + dx, y0 + dy)
            assert [tuple(c) for c in (want - 50000).tolist()] == got, (x0, y0, dx, dy)
    # cells outside a small grid are walked but not counted
    got = [c for c in rr.trace_line(-5, -3, 9, 6) if 0 <= c[0] < 7 and 0 <= c[1] < 5]
    assert [tuple(c) for c in port.trace_line(7, 5, -5, -3, 9, 6).tolist()] == got


@pytest.mark.skipif(not ref.available(), reason="oracle/_ref is not built (SLAM_REFERENCE_DIR)")
def test_karto_trace_line_equals_reference():
    for dx, dy in SEGMENTS + LONG_SEGMENTS[:-1]:
        x0, y0 = max(0, -dx), max(0, -dy)  # the reference allocates the grid: one just big enough for the segment
        want = ref.trace_line(abs(dx) + 1, abs(dy) + 1, x0, y0, x0 + dx, y0 + dy)
        assert [tuple(c) for c in want.tolist()] == rr.trace_line(x0, y0, x0 + dx, y0 + dy), (dx, dy)


def test_gmapping_grid_line_equals_restatement():
    for x0, y0 in ((0, 0), (-7, 11)):
        for dx, dy in SEGMENTS + LONG_SEGMENTS:
            want = port.gmap_grid_line(x0, y0, x0 + dx, y0 + dy)
            got = rr.grid_line((x0, y0), (x0 + dx, y0 + dy))
            assert [tuple(c) for c in want.tolist()] == got, (x0, y0, dx, dy)
            assert got[0] == (x0, y0) and got[-1] == (x0 + dx, y0 + dy) and len(got) == max(abs(dx), abs(dy)) + 1


@pytest.mark.skipif(not ref_gmapping.available(), reason="oracle/_ref is not built (SLAM_REFERENCE_DIR)")
def test_gmapping_grid_line_equals_reference():
    for dx, dy in SEGMENTS + LONG_SEGMENTS:
        want = ref_gmapping.grid_line(0, 0, dx, dy)
        assert [tuple(c) for c in want.tolist()] == rr.grid_line((0, 0), (dx, dy)), (dx, dy)


def test_round_helpers():
    for v, want in ((2.5, 3), (-2.5, -3), (1.5, 2), (-0.0, 0), (0.5, 1), (-0.5, -1), (4503599627370495.5, 4503599627370496)):
        assert rr.c_round(v) == want and rr.karto_round(v) == want, v
    # C round() is exact; Karto's floor(v + 0.5) rounds the largest double below 0.5 up (so does the kernels' kround)
    assert rr.c_round(0.49999999999999994) == 0 and rr.karto_round(0.49999999999999994) == 1
    assert rr.c_round(-0.49999999999999994) == 0 and rr.karto_round(-0.49999999999999994) == -1


KARTO = rc.karto_cases()
UNION_CASES = [k for k, c in KARTO.items() if c.bbox is None]


@pytest.mark.parametrize("name", list(KARTO))
def test_karto_cases_keep_off_half_cells(name):
    assert rc.karto_end_margins(KARTO[name]) >= rc.HALF_CELL_MARGIN


@pytest.mark.parametrize("name", UNION_CASES)
def test_karto_brute_force_equals_restatement(name):
    c = KARTO[name]
    a = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution)
    b = port.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution)
    assert (a["width"], a["height"], a["width_step"]) == (b["width"], b["height"], b["width_step"])
    assert np.array_equal(a["offset"], b["offset"]) and a["cell_visits"] == b["cell_visits"]
    for k in ("passes", "hits", "cells"):
        assert np.array_equal(a[k], b[k]), k


def test_karto_cases_are_what_they_claim():
    for w in (64, 65, 71):
        c = KARTO[f"width{w}"]
        a = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution, bbox=c.bbox)
        assert (a["width"], a["width_step"]) == (w, (w + 7) // 8 * 8)
    for name, dims in (("box7x5", (7, 5)), ("box1x1", (1, 1))):
        c = KARTO[name]
        a = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution, bbox=c.bbox)
        assert (a["width"], a["height"]) == dims and a["cell_visits"] > 0
    c = KARTO["all_beyond_threshold"]
    a = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution)
    assert (a["width"], a["height"], a["cell_visits"]) == (0, 0, 0)
    assert {KARTO[f"n{n}_res{r}"].laser.n_readings for n, r in ((1, 0.05), (4097, 0.25), (16384, 1.0))} == {1, 4097, 16384}


def test_karto_sweep_ties_round_up():
    """the tie beams' end cells: heading 0 rounds (m + 0.5) cells up to m + 1, heading pi rounds -(m + 0.5) to -m"""
    c = KARTO["sweep"]
    a = rr.occupancy_grid(c.laser, c.ranges, c.poses, c.resolution)
    scale = 1.0 / c.resolution
    sx = int(round((c.poses[0, 0] - a["offset"][0]) * scale))
    sy = int(round((c.poses[0, 1] - a["offset"][1]) * scale))
    for s in np.flatnonzero(c.ties[:, 0]):
        m = c.ranges[s, 0] * scale - 0.5
        end = sx + int(m) + 1 if c.poses[s, 2] == 0.0 else sx - int(m)
        assert a["hits"][sy, end] >= 1


def test_karto_range_edges():
    """each reading of the range-edge scans alone in a grid that holds every end point: traced or not, hit or not"""
    nothing, free, hit = (False, False), (True, False), (True, True)
    want = {"range_lt": [nothing, hit, nothing, free, free, hit, free, free] + [nothing] * 6 + [hit],
            "range_eq": [nothing, hit, nothing, free, free, hit, nothing, nothing] + [nothing] * 6 + [hit]}
    for name, expect in want.items():
        c = KARTO[name]
        for i, w in enumerate(expect):
            las = rc.laser(1, c.laser.min_angle + i * c.laser.angular_resolution, 0.0, c.laser.min_range,
                           c.laser.max_range, c.laser.range_threshold)
            a = rr.occupancy_grid(las, c.ranges[:1, i:i + 1], c.poses[:1], c.resolution, bbox=[-10, -10, 10, 10])
            assert (a["cell_visits"] > 0, int(a["hits"].sum()) == 1) == w, (name, i, c.ranges[0, i])


@pytest.mark.parametrize("name", ["sweep", "range_filters", "growth", "msx_lt_width_msy_gt_height",
                                  "odd_half_sizes", "msx_eq_width", "msx_eq_width_plus_1", "defect_row_wrap"])
def test_gmapping_brute_force_equals_restatement(name):
    case = rc.gmap_cases()[name]
    a, b = rr.GMapReference(*case.bounds), port.PortGMap(*case.bounds)
    assert (a.size_x, a.size_y) == (b.size_x, b.size_y)
    for call in case.calls:
        assert rc.gmap_end_margin(case, call) >= rc.HALF_CELL_MARGIN
        kw = dict(laser_xy=call.laser_xy, max_range=call.max_range, max_urange=call.max_urange)
        assert a.compute_map(call.ranges, call.angles, **kw) == b.compute_map(call.ranges, call.angles, **kw) == 0
        for x, y in zip(a.cells(), b.cells()):
            assert np.array_equal(x, y)
    assert np.array_equal(a.ros_map(), b.ros_map())


def test_gmapping_shapes_are_what_they_claim():
    cases = rc.gmap_cases()
    for name, want in (("msx_lt_width_msy_gt_height", (96, 96, 100, 95)), ("odd_half_sizes", (96, 64, 98, 66)),
                       ("msx_eq_width", (128, 64, 128, 64)), ("msx_eq_width_plus_1", (64, 32, 63, 32)),
                       ("defect_row_wrap", (512, 512, 511, 511))):
        xmin, ymin, xmax, ymax, d = cases[name].bounds
        a = rr.GMapReference(*cases[name].bounds)
        assert (a.size_x, a.size_y, int((xmax - xmin) / d), int((ymax - ymin) / d)) == want, name
    assert rr.GMapReference(*cases["odd_half_sizes"].bounds).sx2 % 2 == 1


def test_gmapping_row_wrap_case_has_colliding_cells():
    """in the published 511-wide map, storage cell (511, y) (on the wall) and (0, y + 1) (never seen) share a byte;
    the later write, the wall's, wins in the reference's x-outer loop"""
    case = rc.gmap_cases()["defect_row_wrap"]
    a = rr.GMapReference(*case.bounds)
    call = case.calls[0]
    a.compute_map(call.ranges, call.angles, call.laser_xy, call.max_range, call.max_urange)
    n, v, _, _ = a.cells()
    occ_last = np.where(v[:-1, 511] > 0, np.where(n[:-1, 511] / np.maximum(v[:-1, 511], 1) > 0.25, 100, 0), -1)
    occ_first = np.where(v[1:, 0] > 0, np.where(n[1:, 0] / np.maximum(v[1:, 0], 1) > 0.25, 100, 0), -1)
    differ = np.flatnonzero(occ_last != occ_first)
    assert len(differ) >= 100
    ros = a.ros_map().reshape(-1)
    assert np.array_equal(ros[511 * (differ + 1)], occ_last[differ])


def test_gmapping_out_of_map_changes_nothing():
    b = (-8.0, -8.0, 8.0, 8.0, rc.RES)
    a = rr.GMapReference(*b)
    r, ang = rc.random_beams(b, (0.0, 0.0), 50, seed=1)
    assert a.compute_map(r, ang) == 0
    before = [x.copy() for x in a.cells()]
    assert a.compute_map(np.array([1.0, 128 * rc.RES]), np.array([0.3, 0.0])) == -1
    assert all(np.array_equal(x, y) for x, y in zip(before, a.cells()))
    assert a.compute_map(np.array([127 * rc.RES, 128 * rc.RES]), np.array([0.0, math.pi])) == 0
