"""CPU tests pinning the Hector restatement (oracle/hector_oracle.c, PortHectorProcessor) to the reference processor
(the unmodified lesson4 headers, oracle/_ref/libhector_ref.so; replayed from tests/golden/reference/ where that build
is absent) on the edge cases of tests/hector_cases.py: non-square maps, a robot near two edges of the map, 1, 4 and 8
levels, a map of 12 x 12 cells, scans of 0 ... 4096 points, crafted stamp-order rays and match points on the
interpolation limit.  Poses, Hessians and every cell's log-odds and update index are compared bit for bit (the levels
through digests).

One exception: a stream in which the restatement's pose becomes NaN (a Gauss-Newton step through a singular Hessian)
is not given to the reference.  Its next iteration interpolates at a NaN coordinate, whose (int) conversion is
undefined behaviour in the reference (x86 reads far outside the map); the restatement defines it as the device does."""
import numpy as np
import pytest

import hector_cases as hc
from oracle import port, ref_hector as rh
from reference_record import digest, recording


@pytest.fixture
def rec(request):
    with recording(request, rh.available()) as r:
        yield r


@pytest.mark.parametrize("family", hc.FAMILIES)
@pytest.mark.parametrize("geometry", list(hc.GEOMETRIES))
def test_restatement_equals_reference(geometry, family, rec):
    kw = hc.processor_kw(geometry)
    stream = hc.make_stream(geometry, family)
    compared = 0
    for form in hc.FORMS[family]:
        a = port.PortHectorProcessor(**kw)
        pa, ca, flags = hc.run_stream(a, stream, form)
        if form == "given":
            assert flags.all() and np.array_equal(pa.view(np.int32), stream.hints.view(np.int32))
        if np.isnan(pa).any():
            assert (geometry, family) == ("tall_odd", "interp_edge"), "a new stream reaches a singular Hessian"
            first = int(np.flatnonzero(np.isnan(pa).any(1))[0])
            assert np.isnan(pa[first:]).all() if form == "self" else np.isnan(pa[first]).all()
            a.close()
            continue
        b = rec.proxy(lambda: rh.RefHectorProcessor(**kw), digest=("level",))
        pb, cb, _ = hc.run_stream(b, stream, form)
        assert hc.same_bits(pa, pb), (form, np.flatnonzero((pa != pb).any(1)))
        assert hc.same_bits(ca, cb), form
        for lvl in range(kw["levels"]):
            assert tuple(digest(c) for c in a.level(lvl)) == tuple(b.level(lvl)), (form, lvl)
        compared += 1
        a.close()
    assert compared >= 1


def test_edge_cases_reach_their_edges():
    """The generated cases still reach the edges they are named for."""
    for g in hc.GEOMETRIES:
        sx, sy = hc.GEOMETRIES[g]["size_x"], hc.GEOMETRIES[g]["size_y"]
        kw = hc.processor_kw(g)
        p = port.PortHectorProcessor(**kw)
        hc.run_stream(p, hc.make_stream(g, "stamps"), "given")
        ui = p.level(0)[1]
        assert (ui[:, 0] >= 0).any() and (ui[0, :] >= 0).any() and (ui[:, sx - 1] >= 0).any() and (ui[sy - 1, :] >= 0).any(), g
        s = hc.make_stream(g, "long")
        assert [len(x) for x in s.scans] == list(hc.SINGLE_LENGTHS)
        assert [len(x) for x in hc.make_stream(g, "batch_long").scans] == list(hc.BATCH_LENGTHS)
        e = hc.make_stream(g, "empty")
        assert sum(len(x) == 0 for x in e.scans) == 4
        w = hc.make_stream(g, "walk").hints[:, 2]
        assert (w > 2 * np.pi).any() and (w < -2 * np.pi).any() and (np.abs(w) > 3 * np.pi).sum() >= 4
    assert hc.interp_edge_exact("flat")
    # the robot near the map edge: many of the room's rays end outside the map and are dropped
    p = port.PortHectorProcessor(**hc.processor_kw("edge"))
    hc.run_stream(p, hc.make_stream("edge", "walk"), "given")
    ui = p.level(0)[1]
    assert (ui[:, 0] >= 0).any() and (ui[-1, :] >= 0).any()
    # the 12 x 12 map: 3 x 3 coarsest level, almost every ray leaves it
    p = port.PortHectorProcessor(**hc.processor_kw("tiny"))
    assert p.level(2)[0].shape == (3, 3)
