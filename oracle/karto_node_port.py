"""TEST INFRASTRUCTURE — lesson6's SlamKarto node (lesson6/src/karto_slam.cc: laserCallback, getLaser, addScan,
getOdomPose, updateMap) restated in Python around the library's HOST Mapper.  The Mapper is
b2s_mapper_create_with_matcher with oracle.port.mapper_match_hook (the C restatement's MatchScan), so no device is
needed; maps come from oracle.port.occupancy_grid; tf's LinearMath and roscpp's Time / Duration are restated below
operation by operation in double / integer arithmetic.  tests/test_karto_node_reference.py holds it to the unmodified
node, tests/test_gpu_karto_node.py holds the library's b2s_karto_node_* to it.  Only tests/ and tools/ import it."""
from __future__ import annotations

import ctypes as C
import importlib
import math

import numpy as np

from oracle import port

_PKG = "creating-2d-laser-slam-from-scratch_b200"
abi = importlib.import_module(_PKG + ".abi")
THROTTLED, NO_ODOM, NOT_MOVED, PROCESSED = 0, 1, 2, 3


# ---- tf LinearMath: a transform is (basis rows [3][3], origin [3]) of Python floats
def _rotation(q):
    """Matrix3x3::setRotation"""
    x, y, z, w = q
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return [[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]]


def _quaternion(m):
    """Matrix3x3::getRotation"""
    trace = m[0][0] + m[1][1] + m[2][2]
    t = [0.0] * 4
    if trace > 0.0:
        s = math.sqrt(trace + 1.0)
        t[3] = s * 0.5
        s = 0.5 / s
        t[0] = (m[2][1] - m[1][2]) * s
        t[1] = (m[0][2] - m[2][0]) * s
        t[2] = (m[1][0] - m[0][1]) * s
    else:
        i = (2 if m[1][1] < m[2][2] else 1) if m[0][0] < m[1][1] else (2 if m[0][0] < m[2][2] else 0)
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0)
        t[i] = s * 0.5
        s = 0.5 / s
        t[3] = (m[k][j] - m[j][k]) * s
        t[j] = (m[j][i] + m[i][j]) * s
        t[k] = (m[k][i] + m[i][k]) * s
    return t


def _quat_rpy(roll, pitch, yaw):
    """Quaternion::setRPY (tf::createQuaternionFromRPY)"""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    return [sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy]


def _yaw(q):
    """tf::getYaw: Matrix3x3(q).getRPY, solution 1"""
    m = _rotation(q)
    if abs(m[2][0]) >= 1:
        return 0.0
    pitch = -math.asin(m[2][0])
    c = math.cos(pitch)
    return math.atan2(m[1][0] / c, m[0][0] / c)


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _apply(t, v):
    b, o = t
    return [_dot(v, b[0]) + o[0], _dot(v, b[1]) + o[1], _dot(v, b[2]) + o[2]]


def _mul(a, b):
    """Transform product: basis product through tdotx / tdoty / tdotz, origin a(b.origin)"""
    m1, m2 = a[0], b[0]

    def tdot(c, v):
        return m2[0][c] * v[0] + m2[1][c] * v[1] + m2[2][c] * v[2]
    return [[tdot(0, r), tdot(1, r), tdot(2, r)] for r in m1], _apply(a, b[1])


def _inverse(t):
    b, o = t
    inv = [[b[0][0], b[1][0], b[2][0]], [b[0][1], b[1][1], b[2][1]], [b[0][2], b[1][2], b[2][2]]]
    n = [-o[0], -o[1], -o[2]]
    return inv, [_dot(inv[0], n), _dot(inv[1], n), _dot(inv[2], n)]


def _from_row(r):
    return _rotation([float(r[3]), float(r[4]), float(r[5]), float(r[6])]), [float(r[0]), float(r[1]), float(r[2])]


_IDENTITY = ([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]], [0.0, 0.0, 0.0])


def _to_row(t):
    return list(t[1]) + _quaternion(t[0])


# ---- roscpp Duration
def duration_from_sec(d):
    """ros::Duration::fromSec"""
    sec = math.floor(d)
    nsec = int(round_half_away((d - sec) * 1e9))
    sec += nsec // 1000000000
    return int(sec), nsec % 1000000000


def round_half_away(v):
    """std::round"""
    a = math.floor(abs(v))
    a += 1 if abs(v) - a >= 0.5 else 0
    return a if v >= 0 else -a


def stamp_diff(a, b):
    """Time a - Time b as a normalised (sec, nsec) Duration"""
    sec, nsec = int(np.int32(np.uint32(a[0]))) - int(np.int32(np.uint32(b[0]))), \
        int(np.int32(np.uint32(a[1]))) - int(np.int32(np.uint32(b[1])))
    nsec_part = int(math.fmod(nsec, 1000000000))
    sec_part = sec + int(nsec / 1000000000)
    if nsec_part < 0:
        nsec_part += 1000000000
        sec_part -= 1
    return sec_part, nsec_part


def laser_of(geometry, mount, use_scan_range):
    """getLaser: (b2s_laser, inverted)"""
    base_laser = _from_row(mount)
    lp = _mul(base_laser, _IDENTITY)
    offset = (lp[1][0], lp[1][1], _yaw(_quaternion(lp[0])))
    up = _apply(_inverse(base_laser), [0.0, 0.0, 1 + lp[1][2]])
    f = [float(np.float32(getattr(geometry, k))) for k in ("angle_min", "angle_max", "angle_increment", "range_min",
                                                             "range_max")]
    amin, amax, res, rmin, rmax = f
    thr = rmin if use_scan_range < rmin else (rmax if use_scan_range > rmax else use_scan_range)
    m = int(np.uint32(abi.karto_round((amax - amin) / res)))
    laser = abi.Laser(m, 0, amin, res, rmin, rmax, thr, (C.c_double * 3)(*offset))
    return laser, up[2] <= 0


def ros_payload(grid):
    """updateMap's int8 payload from the restated grid's cells {0 unknown, 100 occupied, 255 free}"""
    c = grid["cells"][:, :grid["width"]]
    out = np.full(c.shape, -1, np.int8)
    out[c == 100] = 100
    out[c == 255] = 0
    return out


class PortKartoNode:
    """One SlamKarto over the library's host Mapper; process() takes consecutive parts of a recording."""

    def __init__(self, params, geometry, mount, solver=None):
        Mapper = importlib.import_module(_PKG + ".mapper").Mapper
        self.prm = params
        self.laser, self.inverted = laser_of(geometry, mount, params.use_scan_range)
        self.n_msg = geometry.n_ranges
        mp = params.mapper
        mp.sequential.range_threshold = mp.loop.range_threshold = self.laser.range_threshold
        self.mapper = Mapper(mp, self.laser, match_fn=port.mapper_match_hook(mp, self.laser))
        if solver is not None:
            self.mapper.set_scan_solver(solver)
        self.interval = duration_from_sec(params.map_update_interval)
        self.laser_count, self.got_map, self.last_map = 0, False, (0, 0)
        self.m2o = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]
        self.readings = []
        self.map_poses = []  # the corrected poses each map was built from

    def update_map(self):
        poses = self.mapper.poses()
        self.map_poses.append(poses)
        g = port.occupancy_grid(self.laser, np.array(self.readings), poses, self.prm.resolution)
        return dict(width=g["width"], height=g["height"], offset=g["offset"], resolution=self.prm.resolution), ros_payload(g)

    def process(self, ranges, stamps, odom):
        m = self.laser.n_readings
        ranges = np.asarray(ranges, np.float32).reshape(-1, self.n_msg)
        S = len(ranges)
        out = dict(state=np.zeros(S, np.int32), pose=np.zeros((S, 3)), map_to_odom=np.zeros((S, 7)),
                   map_published=np.zeros(S, np.int32), maps=[])
        for i in range(S):
            idx = self.laser_count
            self.laser_count += 1
            state = THROTTLED
            if self.laser_count % self.prm.throttle_scans == 0:
                row = np.asarray(odom[i], np.float64)
                if np.isnan(row).any():
                    state = NO_ODOM
                else:
                    ob = _from_row(row)
                    op = _mul(ob, (_rotation(_quat_rpy(0.0, 0.0, 0.0)), [0.0, 0.0, 0.0]))
                    odom_pose = (op[1][0], op[1][1], _yaw(_quaternion(op[0])))
                    r = ranges[i][::-1] if self.inverted else ranges[i]
                    readings = r[:m].astype(np.float64)
                    ok, pose = self.mapper.process(readings, odom_pose, 0.0, sensor="laser")
                    if not ok:
                        state = NOT_MOVED
                    else:
                        state = PROCESSED
                        out["pose"][i] = pose
                        self.readings.append(readings)
                        c = (_rotation(_quat_rpy(0.0, 0.0, float(pose[2]))), [float(pose[0]), float(pose[1]), 0.0])
                        otm = _mul(ob, _inverse(c))
                        self.m2o = _to_row(_inverse((_rotation(_quaternion(otm[0])), otm[1])))
                        st = (int(stamps[i][0]), int(stamps[i][1]))
                        if not self.got_map or stamp_diff(st, self.last_map) > self.interval:
                            info, payload = self.update_map()
                            out["maps"].append((idx, info, payload))
                            out["map_published"][i] = 1
                            self.last_map, self.got_map = st, True
            out["state"][i] = state
            out["map_to_odom"][i] = self.m2o
        return out

    def close(self):
        self.mapper.close()
