"""lesson4's make-map node kernels (csrc/lesson4_node_maps.cu: k_gmn_check, k_gmn_update, k_gmn_publish, k_hmn_free,
k_hmn_occ) against the brute-force node builds (node_maps_reference.py, pinned to the unmodified nodes by
tests/test_node_maps_reference.py) on every crafted call of node_maps_edge_cases.py: every byte of every map, the
refused scan and the untouched output of a refused call.  The Hector maps also equal the map handle's
update_by_scan_just_once + copy_ros on a fresh handle per scan."""
import functools

import numpy as np
import pytest

import node_maps_edge_cases as ec
import node_maps_reference as nr

pytestmark = pytest.mark.gpu

G, H = ec.gmapping_cases(), ec.hector_cases()


@pytest.fixture(scope="module")
def NM(pkg):
    if pkg.load("matcher").device_count() < 1:
        pytest.fail("no CUDA device")
    return pkg.load("node_maps")


@functools.lru_cache(maxsize=None)
def hm_brute(name):
    params, fields, ranges = H[name]
    return nr.hector_node(fields, params, ranges)[0]


def same(got, want, what):
    assert got.shape == want.shape, (got.shape, want.shape)
    for s in range(len(want)):
        bad = np.argwhere(got[s] != want[s])
        assert bad.size == 0, f"{what}: scan {s}: {len(bad)} bytes differ, first (row, col) {bad[:5].tolist()}"


@pytest.mark.parametrize("name", sorted(G))
def test_gmapping_node_maps(NM, pkg, name):
    params, fields, ranges = G[name]
    maps, k, _ = nr.gmapping_node(fields, params, ranges)
    if k == len(ranges):
        same(NM.gmapping_maps(ranges, fields, params), maps, name)
        return
    # the node asserts on scan k: the call names it and writes nothing; the scans before it are mapped
    M, abi = pkg.load("matcher"), pkg.abi
    w, h = nr.gmapping_dims(params)
    out = np.full((len(ranges), h, w), 7, np.int8)
    with pytest.raises(M.B2SError) as e:
        NM.gmapping_maps(ranges, fields, params, out=out)
    assert e.value.status == abi.B2S_ERR_OUT_OF_RANGE and f"scan {k}:" in str(e.value)
    assert (out == 7).all(), "a refused call wrote to the output"
    assert k > 0
    same(NM.gmapping_maps(ranges[:k], fields, params), maps, name)


@pytest.mark.parametrize("name", sorted(H))
def test_hector_node_maps(NM, name):
    params, fields, ranges = H[name]
    same(NM.hector_maps(ranges, fields, params), hm_brute(name), name)


@pytest.mark.parametrize("name", sorted(H))
def test_hector_map_handle(pkg, NM, name):
    """b2s_hector_map_update_by_scan_just_once + b2s_hector_map_copy_ros on a fresh handle per scan, fed the node's
    points"""
    Hm = pkg.load("hector")
    params, fields, ranges = H[name]
    w, h = nr.hector_dims(params)
    want = hm_brute(name)
    for s, r in enumerate(ranges):
        m = Hm.HectorMap(w, h, float(np.float32(params.delta)))
        try:
            m.update_by_scan_just_once(nr.hector_points(fields, r), (0.0, 0.0))
            same(m.ros_map()[None], want[s:s + 1], f"{name} handle scan {s}")
        finally:
            m.close()
