"""The Karto matcher's kernel paths that scans of real rooms never reach, on the device, against two references: the
brute-force integer volume of tests/karto_volume_reference.py and the C restatement (oracle/karto_oracle.c).

Integer volumes are bit-exact against both, results within 1e-9 of the restatement, status and tie counts equal.
The crafted cases and the CPU tests that keep them on their edges are in karto_volume_reference.py.
"""
import numpy as np
import pytest

import karto_volume_reference as kv
from karto_volume_reference import D, abi

pytestmark = pytest.mark.gpu
TOL = 1e-9


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


def handle(M, bt, kernel=0):
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=bt.B, max_base_scans=1)
    m.set_kernel(kernel)
    m.set_scans(bt.ranges, bt.poses)
    m.set_grids(bt.grids, bt.offs)
    return m


def check_batch(m, bt, se, matches=None, cov_in=None, brute=True, exact_xy=False):
    """one CorrelateScan of the whole batch on the device; each listed match against both references"""
    gpu = m.correlate_scan(bt.centers, se, cov_in)
    resp, pose, cov, status, ties = gpu
    dims = (abi.n_steps(se.offset_y, se.res_y), abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.angle_offset, se.angle_res))
    for b in range(bt.B) if matches is None else matches:
        rc, res, sums = bt.oracle(b, se, None if cov_in is None else cov_in[b])
        assert status[b] == rc, (b, status[b], rc)
        if rc:
            continue
        vol = m.response_sums(b, dims)
        assert np.array_equal(vol, sums), b
        if brute:
            assert np.array_equal(vol, bt.brute(b, se)), b
        assert abs(resp[b] - res.response) <= TOL, b
        assert np.allclose(pose[b], res.pose[:], rtol=0, atol=TOL), b
        assert np.allclose(cov[b].ravel(), res.cov[:], rtol=0, atol=TOL), b
        assert ties[b] == res.tie_count, (b, ties[b], res.tie_count)
        if exact_xy:
            assert np.array_equal(pose[b][:2], np.array(res.pose[:2])), b
    return gpu


@pytest.mark.parametrize("geom", kv.PROBE_GEOMS, ids=["small", "banded-12m", "banded-0.025"])
@pytest.mark.parametrize("stride", [1, 2])
def test_probe_grids(M, geom, stride):
    """isolated cells at window corners, block edges, padding columns, both ends of the data, row ends, band seams and
    halo rows; 64 different grids in one launch, on the window kernel with and without empty-window dropping and on the
    generic kernel"""
    bt, se = kv.probe_batch(geom, stride, seed=100 + stride)
    m = handle(M, bt)
    for kernel in (2, 3, 1):
        m.set_kernel(kernel)
        check_batch(m, bt, se, brute=kernel == 2)
        assert m.last_timing()["path"] == min(kernel, 2)
        if kernel == 2:
            assert m.last_stats()["empty_window_frac"] > 0.5  # the sparse grids leave most windows empty
    m.close()


@pytest.mark.parametrize("value", [100, 127])
@pytest.mark.parametrize("n", [2048, 4000, kv.LIST_MAX_BEAMS])
def test_saturated_grids_on_the_window_kernel(M, n, value):
    """every byte 100 or 127 and more than 512 beams per alignment class: the packed-u16 accumulators are flushed
    within a class and come within 511 of overflowing"""
    bt, se = kv.uniform_batch(n, value)
    m = handle(M, bt)
    check_batch(m, bt, se)
    assert m.last_timing()["path"] == 2
    m.close()


def test_beam_count_past_the_list_stage_and_high_bytes(M):
    """7 875 beams are one more than the list stage takes: the generic kernel, and forcing the window kernel is refused.
    Bytes above 127 do not fit the window kernel's packed arithmetic: the generic kernel, with the same numbers."""
    bt, se = kv.uniform_batch(kv.LIST_MAX_BEAMS + 1, 127)
    m = handle(M, bt)
    check_batch(m, bt, se)
    assert m.last_timing()["path"] == 1
    m.set_kernel(2)
    with pytest.raises(M.B2SError) as e:
        m.correlate_scan(bt.centers, se)
    assert e.value.status == abi.B2S_ERR_TOO_LARGE
    m.close()
    for value in (128, 255):
        bt, se = kv.uniform_batch(2048, 100)
        bt.grids[0, ::97] = value
        bt.grids[1, bt.g.data_size // 2] = value
        m = handle(M, bt)
        check_batch(m, bt, se)
        assert m.last_timing()["path"] == 1
        m.close()


@pytest.mark.parametrize("sigma", [10.0, 9.99, 9.98])
def test_degenerate_smear_grids_and_match(M, sigma):
    """smear deviations at the edge where an off-centre kernel value reaches 100 and AddScan depends on the order of
    the points: grid bytes equal to the restatement's, and MatchScan's results too"""
    params, laser_s, cur_r, cur_p, bran, bpos = kv.degenerate_smear_inputs(sigma)
    laser = abi.laser_from(laser_s)
    B, nb = bran.shape[:2]
    m = M.ScanMatcher(params, laser, max_batch=B, max_base_scans=nb)
    for pen in (True, False):
        resp, pose, cov, status, ties = m.match_scan_host(cur_r, cur_p, bran, bpos, pen, True)
        for b in range(B):
            pm = kv.port.PortMatcher(params, laser)
            rc, res = pm.match_scan(cur_r[b], cur_p[b], bran[b], bpos[b], pen, True)
            grid, off = m.grid(b)
            assert np.array_equal(off, pm.grid_off) and np.array_equal(grid, pm.grid), (sigma, b)
            assert status[b] == rc == 0
            assert abs(resp[b] - res.response) <= TOL
            assert np.allclose(pose[b], res.pose[:], rtol=0, atol=TOL)
            assert np.allclose(cov[b].ravel(), res.cov[:], rtol=0, atol=TOL)
    m.close()


@pytest.mark.parametrize("stride", [1, 2])
def test_irregular_lattice_in_a_window_batch(M, stride):
    """a rounding-tie centre (irregular lattice: the window kernel skips it and the generic kernel computes its lookups
    on the fly), an out-of-range centre and regular matches in one batch on the window kernel"""
    bt, se = kv.irregular_batch(stride)
    m = handle(M, bt, kernel=2)
    resp, pose, cov, status, ties = check_batch(m, bt, se)
    assert m.last_timing()["path"] == 2
    assert status[1] == abi.B2S_ERR_OUT_OF_RANGE and (np.delete(status, 1) == 0).all()
    m.close()


@pytest.mark.parametrize("shape", kv.TIE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_tie_counts_around_the_sequential_limit(M, shape):
    """every candidate ties: up to 512 ties the mean x and y are the reference's sequential sums, bit for bit"""
    bt, se = kv.tie_batch(*shape)
    m = handle(M, bt)
    resp, pose, cov, status, ties = check_batch(m, bt, se, exact_xy=np.prod(shape) <= kv.RED_MAX_TIES)
    assert (ties == np.prod(shape)).all()
    m.close()


@pytest.mark.parametrize("na", [1024, 1025])
def test_angle_counts_around_the_penalty_table(M, na):
    """1 024 angles have k_reduce's per-angle float table, 1 025 do not (every candidate evaluated exactly)"""
    bt, se = kv.probe_batch(kv.SMALL, 1, seed=7, B=4)
    rng = np.random.default_rng(na)
    bt.grids[:] = rng.integers(0, 101, size=bt.grids.shape) * (rng.random(bt.grids.shape) < 0.3)
    ar = 0.02 * D
    for pen in (1, 0):
        se = abi.Search(3 * bt.resolution, 3 * bt.resolution, bt.resolution, bt.resolution, 0.5 * (na - 1) * ar, ar, pen, 0)
        assert abi.n_steps(se.angle_offset, se.angle_res) == na
        m = handle(M, bt)
        check_batch(m, bt, se, brute=False)
        m.close()


def test_fine_stage_at_the_angle_limit(M):
    """the fine stage's angular covariance keeps one response per angle in 48 KB: 6 144 angles run, 6 145 are refused"""
    bt, se = kv.probe_batch(kv.SMALL, 1, seed=9, B=2)
    rng = np.random.default_rng(6144)
    bt.grids[:] = rng.integers(0, 101, size=bt.grids.shape)
    r, ar = bt.resolution, 0.005 * D
    cov_in = np.tile(np.eye(3).ravel() * 0.01, (bt.B, 1))
    m = handle(M, bt)
    for na in (6144, 6145):
        se = abi.Search(r, r, r, r, 0.5 * (na - 1) * ar, ar, 1, 1)
        assert abi.n_steps(se.angle_offset, se.angle_res) == na
        if na == 6144:
            check_batch(m, bt, se, cov_in=cov_in, brute=False)
        else:
            with pytest.raises(M.B2SError) as e:
                m.correlate_scan(bt.centers, se, cov_in)
            assert e.value.status == abi.B2S_ERR_TOO_LARGE
    m.close()


def test_responses_at_the_tolerance(M):
    """10 000 beams with 1-3 valid readings: one unit of a sum is 1e-6 of response, so the float pre-filter has to get
    the DoubleEqual tie test and the penalty's zero test right within a unit"""
    bt, se = kv.tolerance_batch()
    for pen in (1, 0):
        se.do_penalize = pen
        m = handle(M, bt)
        check_batch(m, bt, se)
        assert m.last_timing()["path"] == 1  # too many beams for the list stage
        m.close()


def test_add_scans_beyond_add_scan_shared_memory(M, pkg):
    """12 000 beams: more than k_add_scan can stage in shared memory.  The grids are still the restatement's, and so
    are MatchScan's results."""
    synth = pkg.synth
    laser_s = kv.make_laser(12_000, rt=6.0)
    params = abi.matcher_params(1.0, 0.05, 0.03, 6.0)
    laser = abi.laser_from(laser_s)
    world, poses, ranges = synth.make_trajectory(77, 4, laser_s, step_xy=0.08, step_th_deg=2)
    B = 2
    cur_r, cur_p = ranges[2:], poses[2:] + np.array([0.03, -0.02, 0.01])
    bran, bpos = np.stack([ranges[:2]] * B), np.stack([poses[:2]] * B)
    m = M.ScanMatcher(params, laser, max_batch=B, max_base_scans=2)
    resp, pose, cov, status, ties = m.match_scan_host(cur_r, cur_p, bran, bpos)
    for b in range(B):
        pm = kv.port.PortMatcher(params, laser)
        rc, res = pm.match_scan(cur_r[b], cur_p[b], bran[b], bpos[b])
        assert np.array_equal(m.grid(b)[0], pm.grid)
        assert status[b] == rc == 0
        assert abs(resp[b] - res.response) <= TOL and np.allclose(pose[b], res.pose[:], rtol=0, atol=TOL)
        assert np.allclose(cov[b].ravel(), res.cov[:], rtol=0, atol=TOL)
    m.close()
