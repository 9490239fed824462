"""The brute-force node builds of node_maps_reference.py on the crafted calls of node_maps_edge_cases.py (CPU), pinned to
the unmodified nodes (oracle/ref_lesson4, live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere)
and byte for byte to the C restatement (oracle/lesson4_nodes_port), the refused scan included; and the premises that
make each case exercise what it is named for."""
import functools
import math

import numpy as np
import pytest

import lesson4_nodes_cases as lc
import node_maps_edge_cases as ec
import node_maps_reference as nr
from oracle import lesson4_nodes_port as port
from oracle import ref_lesson4
from reference_record import digest, recording

G, H = ec.gmapping_cases(), ec.hector_cases()
CHUNK_BYTES = 256 << 20  # lesson4_node_maps.cu: device memory per stream for one chunk's scratch and payloads


@functools.lru_cache(maxsize=None)
def gm_brute(name):
    params, fields, ranges = G[name]
    return nr.gmapping_node(fields, params, ranges)


@functools.lru_cache(maxsize=None)
def hm_brute(name):
    params, fields, ranges = H[name]
    return nr.hector_node(fields, params, ranges)


def _digests(maps):
    return [digest(m) for m in maps]


@pytest.mark.parametrize("name", sorted(G))
def test_gmapping_brute_force_equals_node(request, name):
    """Every published map and the scan the node asserts on."""
    params, fields, ranges = G[name]
    with recording(request, ref_lesson4.available()) as rec:
        def node():
            maps, k, _, _ = ref_lesson4.gmapping(lc.ros_params(params), fields, ranges)
            return {"maps": _digests(maps), "published": k}
        want = rec.value("gmapping", node, inputs=(name, lc.ros_params(params), ranges))
    maps, k, _ = gm_brute(name)
    assert k == want["published"], f"the brute force refuses scan {k}, the node asserts on scan {want['published']}"
    assert _digests(maps) == list(want["maps"])


@pytest.mark.parametrize("name", sorted(H))
def test_hector_brute_force_equals_node(request, name):
    params, fields, ranges = H[name]
    with recording(request, ref_lesson4.available()) as rec:
        want = rec.value("hector", lambda: _digests(ref_lesson4.hector(lc.ros_params(params), fields, ranges)),
                         inputs=(name, lc.ros_params(params), ranges))
    assert _digests(hm_brute(name)[0]) == list(want)


@pytest.mark.parametrize("name", sorted(G))
def test_gmapping_brute_force_equals_restatement(name):
    params, fields, ranges = G[name]
    maps, k, _ = gm_brute(name)
    got, first, _, _ = port.gmapping(fields, params, ranges)
    assert first == k
    assert np.array_equal(got[:k], maps)


@pytest.mark.parametrize("name", sorted(H))
def test_hector_brute_force_equals_restatement(name):
    params, fields, ranges = H[name]
    assert np.array_equal(port.hector(fields, params, ranges), hm_brute(name)[0])


# ------------------------------------------------------------------------------------------------------- premises


def _visits(scan):
    v = np.zeros(scan.msx * scan.msy, np.int64)
    for (x, y), c in scan.visits.items():
        v[x + y * scan.msx] = c
    return v


@pytest.mark.parametrize("name", ["wrap_right_edge", "wrap_corner"])
def test_wrapped_rows_have_visited_writers(name):
    """W = msx - 1: payload byte (0, y + 1) is written by storage cells (0, y + 1) and then (msx - 1, y).  Many such
    bytes have a visited last writer, some a visited first writer, and publishing the first write instead changes the
    map; visited cells of storage row msy - 1 fall at or past W * H."""
    params, fields, ranges = G[name]
    w, h = nr.gmapping_dims(params)
    scan = gm_brute(name)[2][0]
    assert w == scan.msx - 1
    last, first = nr.gmapping_writers(scan.msx, scan.msy, w, h)
    wrapped = (last != first) & (last >= 0)
    v = _visits(scan)
    n_last, n_first = (wrapped & (v[np.maximum(last, 0)] > 0)).sum(), (wrapped & (v[np.maximum(first, 0)] > 0)).sum()
    assert n_last > 100 and n_first > 0, (n_last, n_first)
    cells = scan.classes(params.occ_thresh)
    assert (nr.gmapping_publish(cells, w, h, last_writer=False) != nr.gmapping_publish(cells, w, h)).sum() > 100
    # free (not only end) cells in the last column, and visited cells in the last row
    assert sum(1 for line in scan.lines for c in line[:-1] if c[0] == scan.msx - 1) > 0
    if name == "wrap_corner":
        assert sum(1 for line in scan.lines for c in line[:-1] if c[1] == scan.msy - 1) > 0


@pytest.mark.parametrize("name, relation", [("exact_storage", 0), ("small_storage", 1)])
def test_storage_contrast_cases(name, relation):
    """W = msx and W > msx: no byte has two writers, and the last storage column is visited."""
    params = G[name][0]
    w, h = nr.gmapping_dims(params)
    scan = gm_brute(name)[2][0]
    assert (w > scan.msx) if relation else (w == scan.msx)
    last, first = nr.gmapping_writers(scan.msx, scan.msy, w, h)
    assert np.array_equal(last, first)
    assert any(x == scan.msx - 1 for (x, _) in scan.visits)


def test_threshold_counters():
    """the laser cell's n and visits at B2S_NODE_MAPS_MAX_RANGES beams, and its published byte (occ_thresh 0.25,
    strictly greater is occupied)"""
    for name, n, visits, byte in (("laser_cell_all", 16384, 16384, 100), ("thresh_equal", 4096, 16384, 0),
                                  ("thresh_over", 4097, 16384, 100)):
        maps, _, (scan,) = gm_brute(name)
        assert G[name][2].shape[1] == ec.FULL
        assert (scan.n[scan.p0], scan.visits[scan.p0]) == (n, visits), name
        assert maps[0, scan.p0[1], scan.p0[0]] == byte, name


def _octant(p0, p1):
    dx, dy = p1[0] - p0[0], p1[1] - p0[1]
    return (dx >= 0, dy >= 0, abs(dx) >= abs(dy))


def test_octant_lines():
    """every octant, walks from p0 and from p1, end points within float steps of a half cell rounding both ways, and
    lines of dmaj 0 and 1 with and without a hit"""
    params, fields, ranges = G["octants"]
    scan = gm_brute("octants")[2][0]
    assert len({_octant(scan.p0, p1) for p1, _ in scan.ends}) == 8
    # gridLine walks from the end with the smaller dominant coordinate (gridlinetraversal.h)
    p0 = scan.p0
    from_p1 = {p0[0] > p1[0] if abs(p1[1] - p0[1]) <= abs(p1[0] - p0[0]) else p0[1] > p1[1] for p1, _ in scan.ends}
    assert from_p1 == {True, False}
    angles = nr.gmapping_angles(fields, ranges.shape[1])
    near = {True: 0, False: 0}
    for i, d in enumerate(ranges[0]):
        d = min(float(d), params.max_use_range)
        for v, c in ((d * math.cos(angles[i]), scan.cx), (d * math.sin(angles[i]), scan.cy)):
            u = (v - c) / params.delta
            if abs(abs(u - math.trunc(u)) - 0.5) < 1e-5:
                near[abs(u - math.trunc(u)) >= 0.5] += 1
    assert near[True] > 8 and near[False] > 8, near
    kinds = {(max(abs(p1[0] - s.p0[0]), abs(p1[1] - s.p0[1])), hit)
             for s in (scan, gm_brute("laser_cell_lines")[2][0]) for p1, hit in s.ends}
    assert {(0, True), (0, False), (1, True), (1, False)} <= kinds


def test_laser_outside_storage():
    """the laser cell lies outside the storage; scan 0 keeps no beam and is mapped, scan 1 keeps one beam whose end
    cell is inside and is refused"""
    params, fields, ranges = G["laser_outside"]
    maps, k, (scan,) = gm_brute("laser_outside")
    assert not scan.inside(scan.p0) and k == 1 and not scan.ends
    assert (maps[0] != 0).any()
    bad = nr.GMappingScan(params, nr.gmapping_angles(fields, ranges.shape[1]), ranges[1])
    assert bad.refused
    kept = [i for i, d in enumerate(ranges[1]) if math.isfinite(d) and 0 < d <= params.max_range]
    assert len(kept) == 1
    a = nr.gmapping_angles(fields, ranges.shape[1])[kept[0]]
    assert bad.inside(bad.world2map(float(ranges[1, kept[0]]) * math.cos(a), float(ranges[1, kept[0]]) * math.sin(a)))


def _crossed(scan):
    """how many drawn end cells an earlier beam's free line crosses, and how many a later one's"""
    first, last = {}, {}
    for b, (_, drawn, freed) in enumerate(scan.beams):
        for o in freed:
            first.setdefault(o, b)
            last[o] = b
    earlier = later = 0
    for b, ((x, y), drawn, _) in enumerate(scan.beams):
        if drawn:
            o = y * scan.width + x
            earlier += first.get(o, b) < b
            later += last.get(o, b) > b
    return earlier, later


def test_hector_comb_crossings():
    """long beams free the end cells of short beams both before and after them in beam order, and a long beam's
    line runs along its own end row"""
    scan = hm_brute("comb")[1][0]
    earlier, later = _crossed(scan)
    assert earlier > 50 and later > 50, (earlier, later)
    assert any(sum(o // scan.width == y for o in freed) > 2 for (x, y), drawn, freed in scan.beams if drawn)
    # the ordered build needs the marks: an end cell freed earlier ends occupied, not free
    maps = hm_brute("comb")[0][0]
    assert all(maps[y, x] == 100 for (x, y), drawn, _ in scan.beams if drawn)


def test_hector_short_beams():
    """end cells on the begin cell (da = 0, not drawn) and one cell away (da = 1), and points within float steps of the
    +-1/2 cell rounding boundary, rounded both ways"""
    params, fields, ranges = H["short_beams"]
    scan = hm_brute("short_beams")[1][0]
    da = [max(abs(x - nr.BEGIN[0]), abs(y - nr.BEGIN[1])) for (x, y), _, _ in scan.beams]
    assert 0 in da and 1 in da
    assert all(len(freed) == 1 for d, (_, drawn, freed) in zip(da, scan.beams) if d == 1)
    ways = set()
    for p in nr.hector_points(fields, ranges[0]):
        for v in p:
            u = abs(float(v) / 0.05)
            if abs(u - 0.5) < 1e-5:
                ways.add(u >= 0.5)
    assert ways == {True, False}


def test_hector_map_edges():
    """drawn end cells on the first and last rows and columns; dropped end cells one beyond each"""
    scan = hm_brute("map_edges")[1][0]
    w, h = scan.width, scan.height
    drawn = [e for e, d, _ in scan.beams if d]
    dropped = [e for e, d, _ in scan.beams if not d]
    assert {0, w - 1} <= {x for x, _ in drawn} and {0, h - 1} <= {y for _, y in drawn}
    assert {-1, w} <= {x for x, _ in dropped} and {-1, h} <= {y for _, y in dropped}
    s801, s800 = hm_brute("begin_last_column")[1][0], hm_brute("begin_outside")[1][0]
    assert (s801.width, s800.width) == (801, 800) and nr.BEGIN[0] == 800
    assert any(d for _, d, _ in s801.beams) and not any(d for _, d, _ in s800.beams)
    assert nr.hector_dims(H["delta_004"][0]) == (2000, 2000)


def test_one_scan_per_chunk():
    """per-scan scratch plus payload above CHUNK_BYTES: every chunk holds one scan"""
    p = G["one_scan_chunks"][0]
    w, h = nr.gmapping_dims(p)
    scan = gm_brute("one_scan_chunks")[2][0]
    assert scan.msx * scan.msy * 4 + w * h > CHUNK_BYTES and scan.msx * scan.msy * 4 == CHUNK_BYTES
    w, h = nr.hector_dims(H["one_scan_chunks"][0])
    assert w * h > CHUNK_BYTES and w > 16384 and h > 16384
    for cases in (G, H):
        _, _, r = cases["one_scan_chunks"]
        assert r.shape == (3, 64)
