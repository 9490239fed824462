"""Angle pruning of the correlative sweep on the device (k_sweep_bound, k_prune_probe, k_prune_select in
csrc/karto_matcher.cu): the results of a pruned CorrelateScan equal the dense sweep's (b2s_matcher_set_kernel(3): every
beam, every angle) bit for bit and the C restatement's within 1e-9, the response volume read back after a pruned call
is the whole dense volume, and on cfg-2 matches most angles are never swept."""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi
from test_prune_bound import walls

pytestmark = pytest.mark.gpu
TOL = 1e-9


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def pruned_and_dense(m, centers, se):
    """one CorrelateScan with automatic selection and one with every angle swept; equal results, byte for byte"""
    m.set_kernel(0)
    auto = m.correlate_scan(centers, se)
    frac = m.last_pruned_frac()
    assert m.last_timing()["path"] == 2
    m.set_kernel(3)
    dense = m.correlate_scan(centers, se)
    assert m.last_pruned_frac() == 0.0
    m.set_kernel(0)
    for a, d in zip(auto, dense):
        assert a.tobytes() == d.tobytes()
    return auto, frac


def assert_matches_restatement(gpu, b, rc, res):
    resp, pose, cov, status, ties = gpu
    assert status[b] == rc, (b, status[b], rc)
    if rc:
        return
    assert abs(resp[b] - res.response) <= TOL, b
    assert np.allclose(pose[b], res.pose[:], rtol=0, atol=TOL), b
    assert np.allclose(cov[b].ravel(), res.cov[:], rtol=0, atol=TOL), b
    assert ties[b] == res.tie_count, (b, ties[b], res.tie_count)


@pytest.mark.parametrize("pen", [1, 0])
def test_cfg2_matches(pkg, M, pen):
    """the benchmark's shape (1081 beams, 31 x 31 x 181, 0.05 m) on seeded synthetic rooms with NaN / inf dropouts"""
    from oracle import port
    synth = pkg.synth
    params, laser = abi.matcher_params(1.5, 0.05, 0.03, 9.25), abi.laser_from(synth.Laser())
    cases = [synth.make_match_case(s, synth.Laser(), dropout=0.02 if s % 4 == 3 else 0.0)
             for s in range(1_000_000, 1_000_008)]
    ranges, poses = np.stack([c.ranges for c in cases]), np.stack([c.odom_pose for c in cases])
    bran, bpos = np.stack([c.base_ranges for c in cases])[:, None, :], np.stack([c.base_pose for c in cases])[:, None, :]
    m = M.ScanMatcher(params, laser, max_batch=len(cases), max_base_scans=1)
    m.set_scans(ranges, poses)
    m.add_scans(bran, bpos)
    se = abi.Search(0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, pen, 0)
    sensor = np.stack([port.PortMatcher(params, laser).sensor_pose(p) for p in poses])
    gpu, frac = pruned_and_dense(m, sensor, se)
    # the dense call came last: sweep the pruned call again, then read its volume back
    m.correlate_scan(sensor, se)
    if pen:
        assert frac >= 0.6, frac  # about 0.88 expected: most angles' bounds lie below best - 0.1
    for b in range(len(cases)):
        pm = port.PortMatcher(params, laser)
        pm.set_scan(ranges[b], poses[b])
        pm.add_scans(bran[b], bpos[b])
        rc, res = pm.correlate_scan(pm.sp, se, want_sums=True)
        assert_matches_restatement(gpu, b, rc, res)
        assert np.array_equal(m.response_sums(b, (31, 31, 181)), pm.last_sums), b
    m.close()


@pytest.mark.parametrize("pen", [1, 0])
def test_crafted_grids_at_the_edges(M, pen):
    """isolated cells at window corners, block edges, padding, both ends of the data and row ends, plus walls along
    every edge of the grid; 41 angles; every match against the restatement, the volume against the brute-force sum"""
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=500, B=32)
    walls(bt, np.random.default_rng(501))
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D, pen=pen)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu, frac = pruned_and_dense(m, bt.centers, se)
    m.correlate_scan(bt.centers, se)
    assert m.last_pruned_frac() == frac
    dims = (abi.n_steps(se.offset_y, se.res_y), abi.n_steps(se.offset_x, se.res_x), 41)
    for b in range(bt.B):
        rc, res, sums = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)
        if rc == 0:
            vol = m.response_sums(b, dims)
            assert np.array_equal(vol, sums), b
            if b % 4 == 0:
                assert np.array_equal(vol, bt.brute(b, se)), b
    m.close()


@pytest.mark.parametrize("pen", [1, 0])
def test_uniform_grid_every_candidate_near_the_best(M, pen):
    """every byte 100: all candidates of an angle tie, so without the penalty nothing may be pruned, and with it only
    angles whose penalty alone puts them 0.1 below the best"""
    bt, _ = kv.uniform_batch(1081, 100, B=3)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=0.5 * D, pen=pen)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu, frac = pruned_and_dense(m, bt.centers, se)
    if not pen:
        assert frac == 0.0
    for b in range(bt.B):
        rc, res, _ = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)
    m.close()


def test_best_below_the_margin_sweeps_every_angle(M):
    """sparse grids whose best response is below 0.1: best - 0.1 <= 0 prunes nothing"""
    bt, _ = kv.probe_batch(kv.SMALL, 1, seed=502, B=16)
    se = kv.window_search(bt, angle_offset=20 * D, angle_res=1 * D)
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    gpu, frac = pruned_and_dense(m, bt.centers, se)
    assert (gpu[0][gpu[3] == 0] < 0.1).all() and frac == 0.0
    for b in range(bt.B):
        rc, res, _ = bt.oracle(b, se)
        assert_matches_restatement(gpu, b, rc, res)
    m.close()
