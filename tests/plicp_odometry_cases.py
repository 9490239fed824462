"""Test streams for the lesson3 odometry node (ScanMatchPLICP, plicp_odometry.cc:191-517) and the helpers every
odometry test shares: the C restatement (orc_plicp_odometry in oracle/plicp_odometry_oracle.c), the unmodified node's
answers (live where oracle/_ref/ is built, replayed from tests/golden/reference/ elsewhere), and packing a run into one
array.

Every stream is a recording of one robot in a synthetic room (synth.py), seeded; the laser is the Hokuyo preset
(1081 beams, -135 .. +135 deg by 0.25 deg, range (0.1, 30) m) with float32 message fields."""
from __future__ import annotations

import importlib
import math

import numpy as np

synth = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.synth")
abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")
plicp = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp")

LASER = synth.Laser()
FIELDS = np.array([LASER.min_angle, LASER.angular_resolution, LASER.min_range, LASER.max_range], np.float32)
IDENTITY = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)


def rpy_quaternion(roll, pitch, yaw):
    """tf2::Quaternion::setRPY as static_transform_publisher builds its message (x, y, z, w)."""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
            cr * cp * cy + sr * sp * sy)


# plicp_odometry.launch: static_transform_publisher args "0 0 0.254 0 0 3.1415926" are x y z yaw pitch roll, so the
# laser is rolled by 3.1415926 (mounted upside down); the same mount read as a yaw of pi is the second one
LAUNCH_MOUNT = (0.0, 0.0, 0.254) + rpy_quaternion(3.1415926, 0.0, 0.0)
YAW_PI_MOUNT = (0.0, 0.0, 0.254) + rpy_quaternion(0.0, 0.0, math.pi)


def cast(world, base_pose, mount, rng, sigma):
    """Ranges of the laser on `mount` with the robot at base_pose: the laser's planar pose in the world and whether
    its scan runs clockwise (a roll of about pi mirrors it)."""
    qx, qy, qz, qw = mount[3:]
    # laser x axis and z axis in base: rows of the rotation matrix of the quaternion
    xx = 1 - 2 * (qy * qy + qz * qz)
    xy = 2 * (qx * qy + qw * qz)
    zz = 1 - 2 * (qx * qx + qy * qy)
    yaw_l = math.atan2(xy, xx)
    c, s = math.cos(base_pose[2]), math.sin(base_pose[2])
    px = base_pose[0] + c * mount[0] - s * mount[1]
    py = base_pose[1] + s * mount[0] + c * mount[1]
    lz = synth.Laser(min_angle=float(FIELDS[0]) * (1 if zz > 0 else -1),
                     angular_resolution=float(FIELDS[1]) * (1 if zz > 0 else -1))
    return synth.cast_scan(world, (px, py, base_pose[2] + yaw_l), lz, rng, sigma)


def stream(seed, steps, dt=0.1, mount=IDENTITY, sigma=0.005, stamps=None, invalid=(), params=None, start=(0, 0, 0)):
    """steps [S][3] = base motion (forward, left, turn in rad) applied before each scan after the first."""
    rng = np.random.default_rng(seed)
    world = synth.make_world(seed)
    pose = np.array(start, np.float64)
    poses, ranges = [], []
    for k in range(len(steps) + 1):
        if k:
            f, l, t = steps[k - 1]
            c, s = math.cos(pose[2]), math.sin(pose[2])
            pose = pose + np.array([c * f - s * l, s * f + c * l, t])
        poses.append(pose.copy())
        ranges.append(cast(world, pose, mount, rng, sigma))
    r = np.array(ranges).astype(np.float32)
    for k in invalid:
        r[k] = 0.0  # no reading above range_min
    if stamps is None:
        t = 1000.0 + dt * np.arange(len(r))
        stamps = np.stack([np.floor(t), np.round((t - np.floor(t)) * 1e9)], 1)
    return dict(ranges=r, stamps=np.asarray(stamps, np.uint32), mount=tuple(mount), poses=np.array(poses),
                params=dict(params or {}))


def _stamps_jitter(n, seed):
    rng = np.random.default_rng(seed)
    ns = 999_900_000 + np.cumsum(rng.integers(40_000_000, 120_000_000, n)) - 40_000_000
    return np.stack([5 + ns // 1_000_000_000, ns % 1_000_000_000], 1)


def _stamps_equal(n, at):
    t = (np.arange(n) * 100_000_000).astype(np.int64)
    t[at] = t[at - 1]
    return np.stack([7 + t // 1_000_000_000, t % 1_000_000_000], 1)


def _streams():
    d = math.radians
    fwd = [(0.03, 0.0, 0.0)] * 30
    out = {
        "straight": stream(1, fwd),
        "rotation": stream(2, [(0.01, 0.0, d(6.5))] * 16),
        "backward": stream(3, [(-0.03, 0.0, 0.0)] * 24),
        "stop_and_go": stream(4, [(0.03, 0, 0)] * 6 + [(0.0, 0, 0)] * 14 + [(0.03, 0, 0)] * 6, sigma=0.0),
        "scan_count": stream(5, [(0.004, 0.0, d(0.2))] * 32),
        "launch_mount": stream(6, [(0.03, 0.0, d(1.0))] * 24, mount=LAUNCH_MOUNT),
        "yaw_pi_mount": stream(7, [(0.03, 0.0, d(-1.0))] * 24, mount=YAW_PI_MOUNT),
        "jitter_stamps": stream(8, [(0.025, 0.005, d(0.5))] * 24, stamps=_stamps_jitter(25, 8)),
        "equal_stamps": stream(9, [(0.02, 0.0, 0.0)] * 12 + [(-0.02, 0.0, 0.0)] * 12, stamps=_stamps_equal(25, 18)),
        "no_valid_reading": stream(10, fwd[:20], invalid=(6, 14)),
        "params": stream(11, [(0.02, 0.0, d(1.5))] * 24,
                         params=dict(kf_dist_linear=0.05, kf_dist_angular=0.04, kf_scan_count=4, max_iterations=6,
                                     outliers_maxPerc=0.8, max_correspondence_dist=0.6, max_angular_correction_deg=30.0,
                                     max_linear_correction=0.5)),
    }
    return out


STREAMS = _streams()


def odom_params(st):
    """b2s_plicp_odom_params of a stream: the node's defaults overridden by its parameter-server values."""
    p = dict(st["params"])
    icp = abi.icp_params(**{k: p.pop(k) for k in list(p) if hasattr(abi.IcpParams, k)})
    return abi.plicp_odom_params(icp=icp, base_to_laser=st["mount"], **p)


def restate(st) -> np.ndarray:
    """orc_plicp_odometry (the C restatement) over a stream -> structured array of plicp.STEP_DTYPE."""
    from oracle import plicp_odometry_port
    return plicp_odometry_port.odometry(odom_params(st), FIELDS, st["ranges"], st["stamps"])


FLOAT_FIELDS = ("position", "orientation", "linear", "angular", "first_guess", "x", "error")
INT_FIELDS = ("valid", "iterations", "nvalid", "published", "keyframe", "reference_scan")


def pack(steps) -> np.ndarray:
    """[S][32] float64: every field of a run (integers widened exactly)."""
    cols = [np.asarray(steps[f], np.float64).reshape(len(steps), -1) for f in FLOAT_FIELDS + INT_FIELDS]
    return np.ascontiguousarray(np.concatenate(cols, 1))


def node_answers(live):
    """{stream name: pack(node run)} from the unmodified node (oracle/ref_lesson3.cpp), live or replayed."""
    from reference_record import Recording
    rec = Recording("test_plicp_odometry_reference__node_streams", live)
    out = {}
    for name, st in STREAMS.items():
        def run(st=st):
            from oracle import ref_lesson3
            return pack(ref_lesson3.run(st["params"], st["mount"], FIELDS, st["ranges"], st["stamps"]))
        out[name] = rec.value(name, run, inputs=(st["ranges"], st["stamps"], list(st["mount"]),
                                                 sorted(st["params"].items())))
    rec.save()
    return out
