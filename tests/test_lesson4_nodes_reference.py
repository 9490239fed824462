"""lesson4's make-map nodes (gmapping.cc, hector_mapping.cc) restated in C (oracle/lesson4_nodes_oracle.c) against the
unmodified nodes (CPU).

The nodes are compiled where they lie against ROS and message stand-ins (oracle/ref_lesson4_*.cpp), live where
oracle/_ref/ is built and from tests/golden/reference/ elsewhere; the maps are compared through digests.  Every line of
the nodes' callbacks that runs is pinned, the GMapping node's writes past the end of its own map included."""
import numpy as np
import pytest

import lesson4_nodes_cases as lc
from oracle import lesson4_nodes_port as port
from oracle import ref_lesson4
from reference_record import digest, recording

G, H = lc.gmapping_cases(), lc.hector_cases()


def _digests(maps):
    return [digest(m) for m in maps]


@pytest.mark.parametrize("name", sorted(G))
def test_gmapping_restatement_equals_node(request, name):
    """Every published byte, the first scan the node asserts on, and the bytes it writes past the end of map_.data."""
    params, fields, ranges = G[name]
    live = ref_lesson4.available()
    with recording(request, live) as rec:
        def node():
            maps, k, ov, nov = ref_lesson4.gmapping(lc.ros_params(params), fields, ranges)
            return {"maps": _digests(maps), "published": k, "overrun": ov, "n_overrun": nov}
        want = rec.value("gmapping", node, inputs=(name, lc.ros_params(params), ranges))
    slack = want["overrun"].shape[1] if want["overrun"].ndim == 2 else 0
    maps, first, ov, nov = port.gmapping(fields, params, ranges, overrun_cap=slack)
    k = want["published"]
    assert first == k, f"the restatement refuses scan {first}, the node asserts on scan {k}"
    assert _digests(maps[:k]) == list(want["maps"])
    assert np.array_equal(ov[:k], want["overrun"]) and np.array_equal(nov[:k], want["n_overrun"])


@pytest.mark.parametrize("name", sorted(H))
def test_hector_restatement_equals_node(request, name):
    params, fields, ranges = H[name]
    live = ref_lesson4.available()
    with recording(request, live) as rec:
        want = rec.value("hector", lambda: _digests(ref_lesson4.hector(lc.ros_params(params), fields, ranges)),
                         inputs=(name, lc.ros_params(params), ranges))
    assert _digests(port.hector(fields, params, ranges)) == list(want)


def test_cases_cover_the_nodes():
    """Each case produces what it is named for."""
    p, f, r = G["room_defaults"]
    maps, first, ov, nov = port.gmapping(f, p, r, overrun_cap=1600)
    assert maps.shape[1:] == (1599, 1599) and port.gmapping_dims(p) == (1599, 1599)
    assert (nov == 1600).all(), "the node's 1 601 writes past the end land on 1 600 bytes"
    assert port.gmapping_dims(G["exact_delta"][0]) == (1280, 1280)
    assert port.gmapping_dims(G["small_storage"][0]) == (999, 999)
    p, f, r = G["leaves_map"]
    assert port.gmapping(f, p, r)[1] == 2, "the small map is not left on scan 2"
    e = G["edges_defaults"][2][0]
    for v in (np.float32(29.99), np.float32(25.0), np.float32(0.1), np.float32(30.0) - np.float32(0.1)):
        assert (e == v).any()
    p, f, r = H["beyond_map"]
    assert (port.hector(f, p, r) == 0).any() and r.max() > 40.0, "no beam ends outside the Hector map"
    p, f, r = H["begin_outside"]
    assert (port.hector(f, p, r) == -1).all()


def test_gmapping_shadowed_column():
    """PublishMap's MAP_IDX(1599, 1599, y) lands on byte (0, y + 1): a hit placed in storage column 1599 shows there."""
    p = lc.node_maps.gmapping_params()
    # one beam along +x to 39.95 m (storage cell x = 800 + 799 = 1599, y = 800), with max ranges wide enough to keep it
    p.max_range, p.max_use_range = 60.0, 50.0
    f = (np.float32(0.0), np.float32(0.01), np.float32(0.1), np.float32(60.0))
    maps, first, _, _ = port.gmapping(f, p, np.array([[39.95]], np.float32))
    assert first == 1 and maps[0, 801, 0] == 100 and maps[0, 800, 1598] == 0


def test_dims_and_refusals_without_device(pkg):
    """The dims query needs no device and equals the restatement's sizing; bad arguments are refused before anything
    else; without a device the maps call is refused with NO_DEVICE (no CPU fallback)."""
    M, abi = pkg.load("matcher"), pkg.abi
    nm = pkg.load("node_maps")
    import ctypes as C
    L = nm._bind()
    for p in (G["room_defaults"][0], G["exact_delta"][0], G["small_storage"][0], G["asymmetric"][0]):
        dims = (C.c_int32 * 2)()
        M.check(L.b2s_gmapping_node_maps(C.byref(nm.geometry(*lc.FIELDS, lc.N)), C.byref(p), 3, None, dims, None, 0,
                                         None))
        assert tuple(dims) == port.gmapping_dims(p)
    for p in (H["room_defaults"][0], H["small_map"][0], H["begin_outside"][0]):
        dims = (C.c_int32 * 2)()
        M.check(L.b2s_hector_mapping_node_maps(C.byref(nm.geometry(*lc.FIELDS, lc.N)), C.byref(p), 3, None, dims, None,
                                               0, None))
        assert tuple(dims) == port.hector_dims(p)
    r = np.zeros((2, nm.MAX_RANGES + 1), np.float32)
    for fn in (nm.gmapping_maps, nm.hector_maps):
        with pytest.raises(M.B2SError) as e:
            fn(r, lc.FIELDS)
        assert e.value.status == abi.B2S_ERR_TOO_LARGE
    with pytest.raises(M.B2SError) as e:
        nm.gmapping_maps(np.zeros((1, 10), np.float32), lc.FIELDS, nm.gmapping_params(xmax=-50.0))
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    with pytest.raises(M.B2SError) as e:
        nm.hector_maps(np.zeros((1, 10), np.float32), lc.FIELDS, nm.hector_params(delta=0.0))
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    if M.device_count() > 0:
        return
    for fn in (nm.gmapping_maps, nm.hector_maps):
        with pytest.raises(M.B2SError) as e:
            fn(G["room_defaults"][2], lc.FIELDS)
        assert e.value.status == abi.B2S_ERR_NO_DEVICE
