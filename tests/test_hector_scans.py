"""Host-only tests of b2s_ros_hector_scans: lesson4's scanCallback conversion of raw LaserScan ranges (laser_geometry's
projectLaser, then rosPointCloudToDataContainer) against the independent restatement in oracle/hector_scans_port.py,
bit for bit, on crafted messages (no GPU)."""
import ctypes as C

import numpy as np
import pytest

from oracle import hector_scans_port as O

f32 = np.float32
AMIN, INC = f32(-2.35619449), f32(0.00436332309619)  # a 1081-beam 270-degree laser


def _up(v):
    return np.nextafter(f32(v), f32(np.inf))


def _down(v):
    return np.nextafter(f32(v), f32(-np.inf))


def _compare(R, ranges, amin=AMIN, inc=INC, rmin=0.1, rmax=30.0, cutoff=30.0, scale=20.0, **filt):
    """The adapter against the restatement; returns the per-scan counts."""
    r = np.asarray(ranges, np.float32)
    r = r.reshape(len(r), -1)
    n = r.shape[1]
    msg = R.make_msg(amin, amin + inc * n, inc, rmin, rmax, np.zeros(n, np.float32))  # (its ranges are ignored)
    pts, cnt, origo = R.hector_scans(msg, r, R.hector_scan_filter(range_cutoff=cutoff, **filt), scale)
    want, worigo = O.scans(r, amin, inc, rmin, rmax, cutoff, scale, **filt)
    assert list(cnt) == [len(w) for w in want]
    cat = np.concatenate(want + [np.zeros((0, 2), np.float32)], 0)
    assert np.array_equal(pts.view(np.int32), cat.view(np.int32))
    assert np.array_equal(origo.view(np.int32), worigo.view(np.int32))
    return cnt


def _walls(n, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.uniform(0.05, 35.0, n)).astype(np.float32)


def test_special_ranges(pkg):
    R = pkg.load("rosio")
    r = _walls(1081)
    r[::7] = np.nan
    r[1::11] = np.inf
    r[2::13] = -np.inf
    r[3::17] = 0.0
    r[4::19] = -2.5
    cnt = _compare(R, r[None])
    finite = np.isfinite(r) & (r >= f32(0.1)) & (r < 30.0)
    assert 0 < cnt[0] <= finite.sum()


def test_range_min_and_cutoff_edges(pkg):
    R = pkg.load("rosio")
    vals = [0.1, _up(0.1), _down(0.1), 30.0, _up(30.0), _down(30.0), 12.3, _up(12.3), _down(12.3)]
    r = np.tile(np.array(vals, np.float32), 40)
    for cutoff in (30.0, 12.3, float(f32(12.3)), 1e9):
        cnt = _compare(R, r[None], rmin=0.1, rmax=30.0, cutoff=cutoff, max_dist=1e4, use_max_scan_range=1e4)
        assert cnt[0] > 0


def test_cutoff_negative_and_above_range_max(pkg):
    R = pkg.load("rosio")
    vals = [7.5, _up(7.5), _down(7.5), 9.0, 11.0, 3.0]
    r = np.tile(np.array(vals, np.float32), 50)
    kw = dict(rmax=7.5, max_dist=100.0, use_max_scan_range=100.0)
    neg = _compare(R, r[None], cutoff=-1.0, **kw)  # -> range_max: 7.5 and above drop out
    above = _compare(R, r[None], cutoff=10.0, **kw)  # used as given, beyond range_max
    assert neg[0] < above[0]


def test_behind_the_robot(pkg):
    R = pkg.load("rosio")
    n = 1440  # a full circle: beams at the back
    inc = f32(2 * np.pi / n)
    r = np.tile(np.array([0.3, 0.6, 0.7, 0.70710677, 0.7071068, 0.75, 1.0], np.float32), n // 7 + 1)[:n]
    cnt = _compare(R, r[None], amin=f32(-np.pi), inc=inc, rmin=0.05)
    assert 0 < cnt[0] < n


def test_use_max_scan_range_edges(pkg):
    R = pkg.load("rosio")
    vals = [20.0, _up(20.0), _down(20.0), 5.5, _up(5.5), _down(5.5), 19.0]
    r = np.tile(np.array(vals, np.float32), 60)
    for use in (20.0, 5.5, float(f32(5.5)) + 1e-12):
        _compare(R, r[None], use_max_scan_range=use)


def test_height_window_without_zero_empties_every_scan(pkg):
    R = pkg.load("rosio")
    r = np.stack([_walls(1081, s) for s in range(3)])
    for z_min, z_max in ((0.1, 1.0), (-1.0, 0.0), (0.0, 1.0)):
        cnt = _compare(R, r, z_min=z_min, z_max=z_max, laser_in_base=(0.1, 0.2, 0.4, 0.3))
        assert not cnt.any(), (z_min, z_max)


@pytest.mark.parametrize("yaw", [0.0, np.pi / 2, -np.pi / 2, 0.7345, -2.9])
def test_laser_pose(pkg, yaw):
    R = pkg.load("rosio")
    r = np.stack([_walls(1081, 10), _walls(1081, 11)])
    cnt = _compare(R, r, laser_in_base=(0.31, -0.17, 0.25, yaw), scale=f32(1.0) / f32(0.05))
    assert cnt.all()


def test_negative_angle_increment(pkg):
    R = pkg.load("rosio")
    r = _walls(1081, 3)
    cnt = _compare(R, r[None], amin=-AMIN, inc=-INC)
    assert cnt[0] > 0


@pytest.mark.parametrize("n", [0, 1, 1081, 4096])
def test_scan_lengths(pkg, n):
    R = pkg.load("rosio")
    r = np.stack([_walls(n, 20 + s) for s in range(2)]) if n else np.zeros((2, 0), np.float32)
    inc = f32(np.deg2rad(270.0) / max(n - 1, 1))
    cnt = _compare(R, r, inc=inc)
    assert len(cnt) == 2 and (cnt.any() or n == 0 or n == 1)


def test_several_scans_per_call(pkg):
    R = pkg.load("rosio")
    r = np.stack([_walls(1081, 30 + s) for s in range(6)])
    r[1] = np.nan  # an all-dropout scan in the middle
    r[4, ::3] = np.inf
    cnt = _compare(R, r, laser_in_base=(0.05, 0.0, 0.1, 0.02))
    assert cnt[1] == 0 and cnt[0] > 0 and cnt[5] > 0


def test_projection_then_existing_filter_equals_adapter(pkg):
    """The restated projection fed into b2s_ros_hector_points gives b2s_ros_hector_scans' points: the refactored
    filter is the one the single-point adapter always applied."""
    R = pkg.load("rosio")
    r = np.stack([_walls(1081, 40 + s) for s in range(3)])
    r[0, ::5] = np.nan
    lb = (0.2, -0.1, 0.3, 0.4)
    kw = dict(min_dist=0.3, max_dist=25.0, use_max_scan_range=18.0, z_min=-0.5, z_max=0.5)
    msg = R.make_msg(AMIN, AMIN + INC * 1081, INC, 0.1, 30.0, np.zeros(1081, np.float32))
    pts, cnt, origo = R.hector_scans(msg, r, R.hector_scan_filter(laser_in_base=lb, range_cutoff=28.0, **kw), 20.0)
    k = 0
    for s in range(3):
        cloud = O.project(r[s], AMIN, INC, 0.1, 30.0, 28.0)
        got, o = R.hector_points(cloud, laser_in_base=lb, scale_to_map=20.0, **kw)
        assert len(got) == cnt[s]
        assert np.array_equal(got.view(np.int32), pts[k:k + cnt[s]].view(np.int32))
        assert np.array_equal(o.view(np.int32), origo.view(np.int32))
        k += cnt[s]
    # caller points with z < 0 or z = -0.0 under a mount at x = y = -0.0: where the rotated sum is exactly -0, tf's
    # z * -0.0 term of the basis makes the coordinate +0.0 (rows 0 and 1), and -0.0 for z > 0 (row 2)
    corner = np.array([[-1.0, -0.0, -0.25], [-0.0, 1.0, -0.0], [-1.0, -0.0, 0.25], [-0.0, 1.0, 0.0]], np.float32)
    for lb in ((-0.0, -0.0, 0.3, 0.0), (0.2, -0.1, 0.3, 0.4)):
        got, o = R.hector_points(corner, laser_in_base=lb, scale_to_map=20.0)
        want, wo = O.to_data_container(corner, lb, 20.0)
        assert len(got) == 4
        assert np.array_equal(got.view(np.int32), want.view(np.int32))
        assert np.array_equal(o.view(np.int32), wo.view(np.int32))
        if lb[0] == 0.0:
            assert list(np.signbit([got[0, 1], got[1, 0], got[2, 1]])) == [False, False, True]


def test_node_defaults_and_bad_arguments(pkg):
    R, M = pkg.load("rosio"), pkg.load("matcher")
    d = R.hector_scan_filter()
    assert (d.range_cutoff, d.use_max_scan_range, d.min_dist, d.max_dist, d.z_min, d.z_max) == (30.0, 20.0, f32(0.2), 30.0, -1.0, 1.0)
    assert C.sizeof(R.HectorScanFilter) == 48
    msg = R.make_msg(AMIN, AMIN, INC, 0.1, 30.0, np.zeros(4, np.float32))
    out, cnt, origo = np.zeros(8, np.float32), np.zeros(1, np.int32), np.zeros(2, np.float32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    L = M.lib()
    R.hector_scans(msg, np.ones((1, 4), np.float32))  # binds the argument types
    r = np.ones(4, np.float32)
    assert L.b2s_ros_hector_scans(C.byref(msg), C.byref(d), 20.0, -1, r.ctypes.data_as(fp), out.ctypes.data_as(fp),
                                  cnt.ctypes.data_as(ip), origo.ctypes.data_as(fp)) == pkg.abi.B2S_ERR_BAD_PARAMS
    assert L.b2s_ros_hector_scans(C.byref(msg), None, 20.0, 1, r.ctypes.data_as(fp), out.ctypes.data_as(fp),
                                  cnt.ctypes.data_as(ip), origo.ctypes.data_as(fp)) == pkg.abi.B2S_ERR_BAD_PARAMS
    assert L.b2s_ros_hector_scans(C.byref(msg), C.byref(d), 20.0, 1, None, out.ctypes.data_as(fp),
                                  cnt.ctypes.data_as(ip), origo.ctypes.data_as(fp)) == pkg.abi.B2S_ERR_BAD_PARAMS
