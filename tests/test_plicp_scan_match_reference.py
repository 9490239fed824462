"""lesson3's scan-to-scan PL-ICP node (ScanMatchPLICP, scan_match_plicp.cc:162-300) restated in C
(orc_plicp_scan_match) against the unmodified node (CPU).

The node is compiled where it lies against ROS and CSM stand-ins (oracle/ref_lesson3_scan_match.cpp), its sm_icp
answered by the PL-ICP restatement, live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere.  Every
line of the node that runs is pinned; sm_icp (CSM) is restated, so it is not."""
import numpy as np
import pytest

import plicp_scan_match_cases as sc
from oracle import ref_lesson3_scan_match


@pytest.fixture(scope="module")
def answers():
    return sc.node_answers(ref_lesson3_scan_match.available())


@pytest.fixture(scope="module")
def restated():
    return {name: sc.restate(st) for name, st in sc.STREAMS.items()}


@pytest.mark.parametrize("name", sorted(sc.STREAMS))
def test_restatement_equals_node(answers, restated, name):
    """valid, iterations, nvalid, x, error and the printed degrees of every scan, bit for bit."""
    mine, node = sc.pack(restated[name]), answers[name]
    same = (mine.view(np.int64) == node.view(np.int64)) | (np.isnan(mine) & np.isnan(node))
    assert same.all(), f"{name}: scan / column {np.argwhere(~same)[0].tolist()} differ from the node"


@pytest.mark.parametrize("switch", sorted(sc.REFUSED))
def test_refused_switch(pkg, answers, switch):
    """A CSM switch the library does not build: the node's stand-in throws, and the parameter helper refuses it."""
    assert answers["refused:" + switch] is True
    with pytest.raises(ValueError):
        pkg.abi.plicp_scan_match_params({switch: 1})
    assert pkg.abi.plicp_scan_match_params({switch: 0}).max_iterations == 10


def test_parameter_helper(pkg):
    """Absent keys keep the node's defaults; the ICP keys set b2s_icp_params; keys the node never reads are refused."""
    abi = pkg.abi
    d, p = abi.icp_params(), abi.plicp_scan_match_params()
    assert bytes(d) == bytes(p)
    p = abi.plicp_scan_match_params(dict(max_iterations=3.0, epsilon_xy=1e-4, outliers_remove_doubles=0, sigma=0.2))
    assert (p.max_iterations, p.epsilon_xy, p.outliers_remove_doubles) == (3, 1e-4, 0)
    with pytest.raises(KeyError):
        abi.plicp_scan_match_params(dict(kf_dist_linear=0.1))


def test_recordings_cover_the_node(restated):
    """Each recording produces the event it is named for."""
    S = restated
    for name, out in S.items():
        assert out["matched"][0] == 0 and (out["matched"][1:] == 1).all(), name
        assert not out["x"][0].any() and out["iterations"][0] == 0, name
    assert len(S["one_scan"]) == 1 and len(S["two_scans"]) == 2 and S["two_scans"]["valid"][1]
    e = sc.STREAMS["edges"]["ranges"]
    lo, hi = sc.LIMITS
    assert (e == lo).any() and (e == hi).any() and np.isnan(e).any() and np.isposinf(e).any() and np.isneginf(e).any()
    lim = np.minimum(sc.STREAMS["limits_change"]["limits"], 1e3)  # finite, so that the differences are
    assert (np.diff(lim[:, 0]) > 0).any() and (np.diff(lim[:, 0]) < 0).any() and (np.diff(lim[:, 1]) < 0).any()
    assert not S["limits_change"]["valid"].all(), "no pair failed on a narrow window"
    same = S["identical"]
    assert (same["valid"][1:] == 1).all() and np.abs(same["x"][1:]).max() < 1e-12, "identical scans did not match"
    assert (same["x"][1:] == same["x"][1]).all(), "identical pairs gave different results"
    big = S["beyond_max_angular"]
    assert not big["valid"][1:].all() and big["valid"][1:].any(), "matches beyond the angular window do not fail"
    assert (S["one_iteration"]["iterations"][1:] == 1).all()
    assert not np.array_equal(S["point_to_point"]["x"], sc.restate(dict(sc.STREAMS["point_to_point"], params={}))["x"])
    assert not np.array_equal(S["keep_doubles"]["nvalid"],
                              sc.restate(dict(sc.STREAMS["keep_doubles"], params={}))["nvalid"])
    nv = S["odom_no_valid_reading"]
    assert not nv["valid"][6] and not nv["valid"][7], "a pair with an empty scan matched"
    deg = np.degrees(S["odom_rotation"]["x"][1:, 2])
    assert np.allclose(S["odom_rotation"]["theta_deg"][1:], deg, rtol=1e-15, atol=0)


def test_create_without_device(pkg):
    """No CPU fallback: without a device create is refused with NO_DEVICE; bad arguments are refused first."""
    P = pkg.load("plicp")
    M = pkg.load("matcher")
    abi = pkg.abi
    amin, ainc = sc.HOKUYO
    for n, a in (([], []), ([2], [amin]), ([1081, 2], [amin, amin])):
        with pytest.raises(M.B2SError) as e:
            P.ScanMatch(abi.icp_params(), n, a, [ainc] * len(a))
        assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    with pytest.raises(M.B2SError) as e:
        P.ScanMatch(abi.icp_params(max_iterations=0), [1081], [amin], [ainc])
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    if M.device_count() > 0:
        return
    with pytest.raises(M.B2SError) as e:
        P.ScanMatch(abi.icp_params(), [1081, 720], [amin, amin], [ainc, ainc])
    assert e.value.status == abi.B2S_ERR_NO_DEVICE
