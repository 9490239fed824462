"""lesson5 motion de-skew (LidarUndistortion): the host preparation of the library against the C restatement (CPU), the
restatement against closed-form motion, and the batched device stage against the restatement (GPU, bit-identical: the two
share an operation order).  The comparison with the unmodified node is tests/test_deskew_reference.py; pcl::getTransformation
and Eigen's Affine3f arithmetic are third-party code absent from the reference tree (see oracle/deskew_oracle.c)."""
import numpy as np
import pytest

from oracle import port
import deskew_cases as dc


def _prepared(pkg, case, use_lib):
    DS = pkg.load("deskew")
    f_imu = DS.integrate_imu if use_lib else port.deskew_integrate_imu
    f_odo = DS.odom_increment if use_lib else port.deskew_odom_increment
    last, t, x, y, z = f_imu(case["imu_stamps"], case["imu_ang"], case["info"].time_start, case["t_end"])
    inc = f_odo(case["start_pose"], case["end_pose"])
    return last, t, x, y, z, inc


def test_host_preparation_equals_restatement(pkg):
    """b2s_deskew_integrate_imu / b2s_deskew_odom_increment (host code of the library, no GPU) vs oracle: same bits."""
    for seed in (1, 2, 3):
        case = dc.make_case(pkg, seed)
        a, b = _prepared(pkg, case, True), _prepared(pkg, case, False)
        assert a[0] == b[0] and a[0] >= 20
        for u, v in zip(a[1:], b[1:]):
            assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    # the node's array bounds: a first message inside the scan would read imu_time_[-1]
    DS = pkg.load("deskew")
    assert DS.integrate_imu([10.0, 10.1], np.zeros((2, 3)), 9.0, 11.0)[0] == -2
    assert port.deskew_integrate_imu([10.0, 10.1], np.zeros((2, 3)), 9.0, 11.0)[0] == -2


def test_restatement_against_closed_form_motion(pkg):
    """Pure yaw at a constant rate: the corrected point of beam i is the measured point turned by yaw(t_i) - yaw(t_first);
    pure translation: shifted by the distance driven since the first valid beam."""
    DS = pkg.load("deskew")
    n = 360
    ranges = np.full(n, 5.0, np.float32)
    ranges[0] = np.inf
    info = DS.DeskewScan()
    info.time_start, info.time_increment, info.range_min, info.range_max = 50.0, 0.1 / n, 0.1, 30.0
    t_end = 50.0 + 0.1 / n * (n - 1)
    a0, da = -np.pi, 2 * np.pi / n
    stamps = 49.99 + np.arange(30) * 0.005
    last, t, x, y, z = port.deskew_integrate_imu(stamps, np.tile([0.0, 0.0, 1.5], (30, 1)), 50.0, t_end)
    info.use_imu, info.use_odom, info.imu_last = 1, 0, last
    out = port.deskew_scan(ranges, a0, da, info, t, x, y, z)
    ti = 50.0 + np.arange(n) * 0.1 / n
    yaw = np.interp(ti, t[:last + 1], z[:last + 1])
    yaw[ti > t[last]] = z[last]
    ang = a0 + np.arange(n) * da + (yaw - yaw[1])
    assert np.all(out[0] == 0) and np.abs(out[1:, 0] - 5 * np.cos(ang[1:])).max() < 2e-5
    assert np.abs(out[1:, 1] - 5 * np.sin(ang[1:])).max() < 2e-5 and np.abs(out[1:, 2] - 1.0).max() < 1e-6
    info.use_imu, info.use_odom = 0, 1
    info.odom_start_time, info.odom_end_time = 49.98, 50.12
    inc = port.deskew_odom_increment([0, 0, 0, 0, 0, 0], [0.14, 0.0, 0.0, 0, 0, 0])
    info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = inc
    out = port.deskew_scan(ranges, a0, da, info, t, x, y, z)
    shift = (ti - ti[1]) * 1.0  # 0.14 m in 0.14 s
    assert np.abs(out[1:, 0] - (5 * np.cos(a0 + np.arange(1, n) * da) + shift[1:])).max() < 2e-5


@pytest.mark.gpu
def test_device_stage_equals_restatement(pkg):
    """Batched CorrectLaserScan on the device (32 scans of 1081 beams with dropouts, IMU + odometry) vs the C restatement:
    identical float bit patterns; IMU-only, odometry-only and no-correction variants included."""
    DS = pkg.load("deskew")
    assert pkg.load("matcher").device_count() > 0
    cases, infos, tabs = [], [], []
    for b in range(32):
        case = dc.make_case(pkg, 100 + b, rate=(0.3 * (b % 3), -0.2, 0.9 + 0.05 * b), vel=(0.5 + 0.02 * b, 0.1, 0.0))
        last, t, x, y, z, inc = _prepared(pkg, case, True)
        info = case["info"]
        info.imu_last = last
        info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = inc
        info.use_imu, info.use_odom = (1, 1) if b % 4 < 2 else ((1, 0) if b % 4 == 2 else (0, 1))
        if b == 31:
            info.use_imu = info.use_odom = 0
        cases.append(case); infos.append(info); tabs.append((t, x, y, z))
    ranges = np.stack([c["ranges"] for c in cases])
    T, X, Y, Z = (np.stack([tb[k] for tb in tabs]) for k in range(4))
    got = DS.undistort(ranges, cases[0]["angle_min"], cases[0]["angle_increment"], infos, T, X, Y, Z)
    for b in range(32):
        want = port.deskew_scan(ranges[b], cases[0]["angle_min"], cases[0]["angle_increment"], infos[b], *tabs[b])
        assert np.array_equal(got[b].view(np.int32), want.view(np.int32)), (b, np.abs(got[b] - want).max())
    valid = np.isfinite(ranges) & (ranges >= 0.1) & (ranges <= 30.0)
    assert np.all(got[~valid] == 0) and np.abs(got[valid]).max() > 1.0
    raw = np.stack([ranges[31] * np.cos(cases[0]["angle_min"] + np.arange(1081) * cases[0]["angle_increment"]),
                    ranges[31] * np.sin(cases[0]["angle_min"] + np.arange(1081) * cases[0]["angle_increment"])], 1)
    v31 = valid[31]
    assert np.abs(got[31][v31, :2] - raw[v31]).max() < 1e-5  # nothing to correct: the measured points


def test_undistort_rejects_bad_arguments_before_touching_a_device(pkg):
    """Argument errors are reported as B2S_ERR_BAD_PARAMS whether or not a GPU is present (imu_last outside the table,
    an odometry interval of zero length, empty scans)."""
    DS, M, abi = pkg.load("deskew"), pkg.load("matcher"), pkg.abi
    case = dc.make_case(pkg, 7, n=64)
    info = case["info"]
    tabs = [np.zeros((1, 16))] * 4
    info.imu_last = 16  # one past the table
    with pytest.raises(M.B2SError) as e:
        DS.undistort(case["ranges"][None, :], case["angle_min"], case["angle_increment"], [info], *tabs)
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    info.imu_last = 3
    info.odom_start_time = info.odom_end_time = 5.0
    with pytest.raises(M.B2SError) as e:
        DS.undistort(case["ranges"][None, :], case["angle_min"], case["angle_increment"], [info], *tabs)
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS


def test_odometry_increment_is_the_relative_pose_in_the_start_frame(pkg):
    """transBegin.inverse() * transEnd (:320-327): the translation of the end pose expressed in the start frame — checked
    against double-precision rotation matrices built independently (roll, pitch, yaw about x, y, z; R = Rz Ry Rx)."""
    DS = pkg.load("deskew")

    def rot(r, p, y):
        cx, sx, cy, sy, cz, sz = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
        rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
        ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
        return rz @ ry @ rx

    rng = np.random.default_rng(4)
    for _ in range(50):
        a = np.concatenate([rng.uniform(-5, 5, 3), rng.uniform(-0.4, 0.4, 2), rng.uniform(-3, 3, 1)])
        b = a + np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])
        want = rot(*a[3:]).T @ (b[:3] - a[:3])
        for got in (DS.odom_increment(a, b), port.deskew_odom_increment(a, b)):
            assert np.abs(got - want).max() < 5e-6, (got, want)
    assert np.array_equal(DS.odom_increment([1, 2, 3, 0, 0, 0], [1.5, 2.25, 3, 0, 0, 0]), np.array([0.5, 0.25, 0.0], np.float32))
