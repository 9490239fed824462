"""lesson3's odometry node with a laser, mount, parameter set and range fields of each recording's own
(plicp_odometry_fleet_cases.py) restated on the CPU against the unmodified node, every LaserScan carrying its own
range fields.

The restatement is orc_plicp_odometry on the scans NaN-masked by their own fields with fields (-inf, inf); the node is
compiled where it lies (oracle/ref_lesson3.cpp), live where oracle/_ref/ is built and replayed from
tests/golden/reference/ elsewhere."""
import numpy as np
import pytest

import plicp_odometry_cases as pc
import plicp_odometry_fleet_cases as fc
from oracle import ref_lesson3


@pytest.fixture(scope="module")
def answers():
    return fc.node_answers(ref_lesson3.available())


@pytest.fixture(scope="module")
def restated():
    return {name: fc.restate(st) for name, st in fc.STREAMS.items()}


def _bits_equal(a, b):
    return ((a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))).all()


@pytest.mark.parametrize("name", sorted(fc.STREAMS))
def test_restatement_equals_node(answers, restated, name):
    """Every published pose, quaternion, twist, first guess, sm_icp result and key-frame decision, bit for bit."""
    mine, node = pc.pack(restated[name]), answers[name]
    same = (mine.view(np.int64) == node.view(np.int64)) | (np.isnan(mine) & np.isnan(node))
    assert same.all(), f"{name}: scan / column {np.argwhere(~same)[0].tolist()} differ from the node"


@pytest.mark.parametrize("name", sorted(pc.STREAMS))
def test_masked_restatement_equals_the_uniform_one(name):
    """On every existing stream (one laser, constant fields) masking each scan by its fields and matching with
    (-inf, inf) gives orc_plicp_odometry's own answers bit for bit."""
    st = fc.all_streams()[name]
    assert _bits_equal(pc.pack(fc.restate(st)), pc.pack(fc.restate_uniform(st)))


def test_streams_cover_their_events(restated):
    """Each stream produces the event it is named for."""
    S, R = fc.STREAMS, restated

    def fields_matter(name):  # the per-scan fields change the answers against constant fields
        return not _bits_equal(pc.pack(R[name]), pc.pack(fc.restate_uniform(S[name])))

    r = S["range_max_drop"]
    assert ((r["ranges"][6:10] > 4.0) & (r["ranges"][6:10] < 30.0)).any() and fields_matter("range_max_drop")
    r = S["range_min_raise"]
    assert ((r["ranges"][8:12] > 0.1) & (r["ranges"][8:12] < 4.0)).any() and fields_matter("range_min_raise")
    r, o = S["keyframe_fields"], R["keyframe_fields"]
    ks = [k for k in range(len(o)) if o[k]["published"] and o[k]["reference_scan"] == 0]
    assert len(ks) >= 3 and all((r["limits"][k] != r["limits"][0]).any() for k in ks), "no match against a key frame " \
        "taken under other fields"
    assert ((r["ranges"][0] > 5.0) & (r["ranges"][0] < 30.0)).any() and fields_matter("keyframe_fields")
    r, o = S["fields_after_promotion"], R["fields_after_promotion"]
    after = [k for k in range(1, len(o)) if o[k - 1]["keyframe"] and (r["limits"][k] != r["limits"][k - 1]).any()]
    assert after == [5, 13], after
    assert fields_matter("fields_after_promotion")
    beams = {st["laser"][0]: st for st in S.values()}
    assert {3, 4, 360, 720, 1081, 1440, 2048, 2408} <= set(beams)
    for n, fov in ((360, 360), (720, 360), (720, 270), (2048, 360), (2408, 270)):
        assert any(st["laser"] == fc.laser(n, fov) for st in S.values()), (n, fov)
    assert all(R[name]["published"][1:].all() and not R[name]["valid"].any() for name in ("laser_3", "laser_4"))
    assert all(R[name]["valid"][1:].all() for name in S if name not in ("laser_3", "laser_4"))
    mounts = {st["mount"] for st in S.values()}
    params = {tuple(sorted(st["params"].items())) for st in S.values()}
    assert len(mounts) >= 3 and len(params) >= 4
