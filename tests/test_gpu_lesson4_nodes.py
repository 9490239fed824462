"""lesson4's make-map nodes on the device (b2s_gmapping_node_maps, b2s_hector_mapping_node_maps) against the C
restatement (oracle/lesson4_nodes_oracle.c, itself pinned to the unmodified nodes by
tests/test_lesson4_nodes_reference.py): every byte of every map, on every case of tests/lesson4_nodes_cases.py, on
long recordings, chunked calls, the beam-count limit and refused calls."""
import ctypes as C

import numpy as np
import pytest

import lesson4_nodes_cases as lc
from oracle import lesson4_nodes_port as port

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def NM(pkg):
    NM, M = pkg.load("node_maps"), pkg.load("matcher")
    if M.device_count() < 1:
        pytest.fail("no CUDA device")
    return NM


def same(got, want, what):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.flatnonzero((got != want).reshape(len(got), -1).any(axis=1))
    assert bad.size == 0, f"{what}: scans {bad[:10]} differ"


def gm(NM, params, fields, ranges):
    maps, first, _, _ = port.gmapping(fields, params, ranges)
    assert first == len(ranges), f"the restatement refuses scan {first}"
    same(NM.gmapping_maps(ranges, fields, params), maps, "GMapping")
    return maps


def hm(NM, params, fields, ranges):
    maps = port.hector(fields, params, ranges)
    same(NM.hector_maps(ranges, fields, params), maps, "Hector")
    return maps


@pytest.mark.parametrize("name", sorted(n for n in lc.gmapping_cases() if n != "leaves_map"))
def test_gmapping_cases(NM, name):
    gm(NM, *lc.gmapping_cases()[name])


@pytest.mark.parametrize("name", sorted(lc.hector_cases()))
def test_hector_cases(NM, name):
    hm(NM, *lc.hector_cases()[name])


def test_gmapping_refuses_rays_leaving_the_map(NM, pkg):
    """The node asserts on scan 2: the call names it and writes nothing."""
    M, abi = pkg.load("matcher"), pkg.abi
    params, fields, ranges = lc.gmapping_cases()["leaves_map"]
    assert port.gmapping(fields, params, ranges)[1] == 2
    out = np.full((len(ranges),) + port.gmapping_dims(params)[::-1], 7, np.int8)
    with pytest.raises(M.B2SError) as e:
        NM.gmapping_maps(ranges, fields, params, out=out)
    assert e.value.status == abi.B2S_ERR_OUT_OF_RANGE and "scan 2:" in str(e.value)
    assert (out == 7).all(), "a refused call wrote to the output"
    # the scans before it are mapped
    gm(NM, params, fields, ranges[:2])


@pytest.mark.parametrize("scans", [1, 2, 1000])
def test_recording_lengths(NM, scans):
    """1, 2 and 1000 scans of a drifting room.  The 1000-scan recording uses 40 m maps (about 0.64 MB per scan); the
    Hector one keeps its fixed begin cell (800, 800) inside with 802 cells."""
    r = lc.recording(20 + scans, scans, (6.0, 4.0), shift_step=(0.002, 0.001))
    if scans < 1000:
        gm(NM, lc.node_maps.gmapping_params(), lc.FIELDS, r)
        hm(NM, lc.node_maps.hector_params(), lc.FIELDS, r)
    else:
        gm(NM, lc.node_maps.gmapping_params(xmin=-20.0, ymin=-20.0, xmax=20.0, ymax=20.0), lc.FIELDS, r)
        hm(NM, lc.node_maps.hector_params(xmin=-20.0, ymin=-20.0, xmax=20.1, ymax=20.1), lc.FIELDS, r)


def test_chunked_calls_equal_one_call(NM):
    r = lc.recording(31, 7, (6.0, 4.0))
    for fn in (NM.gmapping_maps, NM.hector_maps):
        one = fn(r, lc.FIELDS)
        parts = np.concatenate([fn(r[:3], lc.FIELDS), fn(r[3:4], lc.FIELDS), fn(r[4:], lc.FIELDS)])
        assert np.array_equal(one, parts)
        assert fn(r[:0], lc.FIELDS).shape == (0,) + one.shape[1:]


def test_beam_count_limit(NM, pkg):
    """1 beam and B2S_NODE_MAPS_MAX_RANGES beams run; one more is refused and leaves the output untouched."""
    M, abi = pkg.load("matcher"), pkg.abi
    one = lc.recording(41, 2, (6.0, 4.0), n=1)
    gm(NM, lc.node_maps.gmapping_params(), lc.FIELDS, one)
    hm(NM, lc.node_maps.hector_params(), lc.FIELDS, one)
    inc = np.float32(2 * np.pi / NM.MAX_RANGES)
    fields = (np.float32(-np.pi), inc) + lc.FIELDS[2:]
    cap = np.stack([lc._box((6.0, 4.0), NM.MAX_RANGES, angle_min=fields[0], inc=inc)] * 2).astype(np.float32)
    gm(NM, lc.node_maps.gmapping_params(), fields, cap)
    hm(NM, lc.node_maps.hector_params(), fields, cap)
    over = np.zeros((1, NM.MAX_RANGES + 1), np.float32)
    for fn in (NM.gmapping_maps, NM.hector_maps):
        out = np.full((1, 1599, 1599), 7, np.int8)
        with pytest.raises(M.B2SError) as e:
            fn(over, fields, out=out)
        assert e.value.status == abi.B2S_ERR_TOO_LARGE and (out == 7).all()


def test_hector_equals_map_handle(NM, pkg):
    """Each Hector payload also equals b2s_hector_map_update_by_scan_just_once + b2s_hector_map_copy_ros on a fresh
    1599 x 1599 handle per scan, fed the node's points."""
    Hm = pkg.load("hector")
    params, fields, ranges = lc.hector_cases()["hall_defaults"]
    got = NM.hector_maps(ranges, fields, params)
    for s, r in enumerate(ranges):
        angle, pts = np.float32(fields[0]), []
        for d in r:  # ROSLaserScanToDataContainer (hector_mapping.cc:144-163)
            if d > fields[2] and d < np.float32(fields[3]) - np.float32(0.1):
                pts.append((np.float32(np.cos(np.float64(angle)) * np.float64(d)),
                            np.float32(np.sin(np.float64(angle)) * np.float64(d))))
            angle = np.float32(angle + fields[1])
        h = Hm.HectorMap(1599, 1599, 0.05)
        h.update_by_scan_just_once(np.array(pts, np.float32), (0.0, 0.0))
        assert np.array_equal(h.ros_map().reshape(1599, 1599), got[s]), f"scan {s}"
        h.close()


def test_dims_query_and_pinned_output(NM):
    """A NULL output only sizes the payload; a page-locked output buffer receives the same maps as pageable memory."""
    import torch
    r = lc.recording(51, 5, (6.0, 4.0))
    want = NM.gmapping_maps(r, lc.FIELDS)
    pinned = torch.empty(want.shape, dtype=torch.int8, pin_memory=True)
    got = NM.gmapping_maps(r, lc.FIELDS, out=pinned.numpy())
    assert np.array_equal(got, want)
    L = NM._bind()
    dims = (C.c_int32 * 2)()
    assert L.b2s_hector_mapping_node_maps(C.byref(NM.geometry(*lc.FIELDS, lc.N)), C.byref(NM.hector_params()), 5,
                                          None, dims, None, 0, None) == 0 and tuple(dims) == (1599, 1599)
