"""TEST INFRASTRUCTURE — restatement of lesson4's HectorMappingRos node (lesson4/src/hector_mapping/hector_slam.cc) over a
recording, written independently of the library:

  InitParams' squared thresholds            hector_slam.cc:150-155  (squared in double, rounded to float)
  projectLaser                              oracle/hector_scans_port.project (laser_geometry's rule, DESIGN.md §7)
  rosPointCloudToDataContainer              hector_slam.cc:320-362 with the mount's full tf::Transform (setRotation of
                                            its quaternion; operator* row by row, in double)
  HectorSlamProcessor::update               oracle/port.PortHectorProcessor (the C restatement, hector_oracle.c)
  PoseInfoContainer::update + poseMsgToTF   util/PoseInfoContainer.h:53-92
  setMapInfo / publishMap and its gate      hector_slam.cc:165-180, 269-317
  the publish schedule                      the library's definition (include/b200slam.h, DESIGN.md §7)

Double arithmetic is Python's float, transcendental functions are math's (the C library's), float32 steps are numpy
float32 scalar operations."""
from __future__ import annotations

import math

import numpy as np

from oracle import hector_scans_port as scans_port
from oracle import port

f32 = np.float32
NS = 1_000_000_000


def sqr_threshold(metres):
    """p_sqr_laser_min_dist_ = static_cast<float>(tmp * tmp): squared in double, then rounded."""
    return f32(float(metres) * float(metres))


def duration_from_sec(d):
    """ros::Duration::fromSec -> (sec, nsec)."""
    sec = int(math.floor(d))
    x = (d - sec) * 1e9  # >= 0: C's round() is floor, plus one from a fraction of one half up
    nsec = int(math.floor(x))
    if x - nsec >= 0.5:
        nsec += 1
    sec += nsec // NS
    nsec %= NS
    return sec, nsec


class Schedule:
    """The publish schedule: tick 0 = the first scan's stamp, tick k = tick 0 + k * Duration::fromSec(period) (roscpp
    Time + Duration, normalised (sec, nsec)).  before(stamp) -> the tick published before that scan, or None."""

    def __init__(self, period):
        self.period = duration_from_sec(period)
        self.next = None

    def _add(self, t, k):
        sec = t[0] + k * self.period[0]
        nsec = t[1] + k * self.period[1]
        return sec + nsec // NS, nsec % NS

    def before(self, stamp):
        s = (int(stamp[0]) + int(stamp[1]) // NS, int(stamp[1]) % NS)
        if self.next is None:
            self.next = s
        if s < self.next:
            return None
        tick = self.next
        p = self.period[0] * NS + self.period[1]
        d = (s[0] - tick[0]) * NS + (s[1] - tick[1])
        self.next = self._add(tick, d // p + 1)  # the first tick strictly after the stamp
        return tick


def set_rotation(q):
    """tf::Matrix3x3::setRotation."""
    x, y, z, w = (float(v) for v in q)
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return [[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]]


def get_rotation(m):
    """tf::Matrix3x3::getRotation -> (x, y, z, w)."""
    trace = m[0][0] + m[1][1] + m[2][2]
    q = [0.0, 0.0, 0.0, 0.0]
    if trace > 0.0:
        s = math.sqrt(trace + 1.0)
        q[3] = s * 0.5
        s = 0.5 / s
        q[0] = (m[2][1] - m[1][2]) * s
        q[1] = (m[0][2] - m[2][0]) * s
        q[2] = (m[1][0] - m[0][1]) * s
    else:
        i = (2 if m[1][1] < m[2][2] else 1) if m[0][0] < m[1][1] else (2 if m[0][0] < m[2][2] else 0)
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0)
        q[i] = s * 0.5
        s = 0.5 / s
        q[3] = (m[k][j] - m[j][k]) * s
        q[j] = (m[j][i] + m[i][j]) * s
        q[k] = (m[k][i] + m[i][k]) * s
    return q


def to_data_container(pts_xyz, mount, scale_to_map, min_dist=0.2, max_dist=30.0, use_max_scan_range=20.0, z_min=-1.0,
                      z_max=1.0):
    """rosPointCloudToDataContainer with the mount (x, y, z, qx, qy, qz, qw) as the node's laserTransform_."""
    basis, origin = set_rotation(mount[3:]), [float(v) for v in mount[:3]]
    sqr_min, sqr_max = sqr_threshold(min_dist), sqr_threshold(max_dist)
    use = float(use_max_scan_range)
    zmin, zmax, scale = f32(z_min), f32(z_max), f32(scale_to_map)
    out = []
    with np.errstate(all="ignore"):
        for x, y, z in np.asarray(pts_xyz, np.float32).reshape(-1, 3):
            d = x * x + y * y
            if not (d > sqr_min and d < sqr_max):
                continue
            if x < f32(0.0) and d < f32(0.5):
                continue
            if float(d) > use * use:
                continue
            v = (float(x), float(y), float(z))
            b = [basis[r][0] * v[0] + basis[r][1] * v[1] + basis[r][2] * v[2] + origin[r] for r in range(3)]
            zl = f32(b[2] - origin[2])
            if zl > zmin and zl < zmax:
                out.append((f32(b[0]) * scale, f32(b[1]) * scale))
        origo = np.array([f32(origin[0]) * scale, f32(origin[1]) * scale], np.float32)
    return np.array(out, np.float32).reshape(-1, 2), origo


def map_info(resolution, size, start_x, start_y):
    """setMapInfo of level 0: getWorldCoords(0, 0) - cell length * 0.5f, through the Affine2f inverse."""
    cl = f32(resolution)
    off_x, off_y = (cl * f32(size)) * f32(start_x), (cl * f32(size)) * f32(start_y)
    tw = f32(1.0) / cl
    tx, ty = tw * off_x, tw * off_y
    invdet = f32(1.0) / (tw * tw - f32(0.0) * f32(0.0))
    i01 = f32(-0.0) * invdet
    wt = tw * invdet
    wx = (wt * f32(0.0) + f32(-0.0) * f32(0.0)) + (-(wt * tx + i01 * ty))
    wy = (f32(-0.0) * f32(0.0) + wt * f32(0.0)) + (-(i01 * tx + wt * ty))
    return dict(origin_x=float(wx - cl * f32(0.5)), origin_y=float(wy - cl * f32(0.5)), resolution=float(cl),
                width=int(size), height=int(size))


def pose_message(pose, hessian):
    """PoseInfoContainer::update: the pose (x, y, z, qx, qy, qz, qw), the 36 covariance entries and the odom ->
    base_link tf poseMsgToTF makes of it (translation + getRotation of setRotation(q))."""
    half = f32(pose[2]) * f32(0.5)
    msg = [float(f32(pose[0])), float(f32(pose[1])), 0.0, 0.0, 0.0, math.sin(float(half)), math.cos(float(half))]
    h = np.asarray(hessian, np.float32).reshape(3, 3)
    cov = [0.0] * 36
    cov[0], cov[7], cov[35] = float(h[0, 0]), float(h[1, 1]), float(h[2, 2])
    cov[1] = cov[6] = float(h[0, 1])
    cov[5] = cov[30] = float(h[0, 2])
    cov[11] = cov[31] = float(h[1, 2])
    tf = msg[:3] + get_rotation(set_rotation(msg[3:]))
    return msg, cov, tf


class HectorNodePort:
    """One HectorMappingRos over parts of a recording.  params: a dict of InitParams' values (node defaults for absent
    keys); geometry: (angle_min, angle_increment, range_min, range_max)."""

    DEFAULTS = dict(map_resolution=0.05, map_size=2048, map_start_x=0.5, map_start_y=0.5, map_multi_res_levels=3,
                    update_factor_free=0.4, update_factor_occupied=0.9, map_update_distance_thresh=0.4,
                    map_update_angle_thresh=0.9, use_max_scan_range=20.0, laser_min_dist=0.2, laser_max_dist=30.0,
                    laser_z_min_value=-1.0, laser_z_max_value=1.0, map_pub_period=2.0)

    def __init__(self, params: dict, geometry, mount=(0, 0, 0, 0, 0, 0, 1)):
        p = dict(self.DEFAULTS, **params)
        self.p, self.geometry, self.mount = p, tuple(geometry), tuple(float(v) for v in mount)
        res = float(f32(p["map_resolution"]))
        self.proc = port.PortHectorProcessor(res, p["map_size"], p["map_size"], (p["map_start_x"], p["map_start_y"]),
                                             p["map_multi_res_levels"], p["update_factor_free"],
                                             p["update_factor_occupied"], p["map_update_distance_thresh"],
                                             p["map_update_angle_thresh"])
        self.scale = f32(1.0) / f32(res)
        self.info = map_info(res, p["map_size"], p["map_start_x"], p["map_start_y"])
        self.schedule = Schedule(p["map_pub_period"])
        self.scans, self.update_index, self.last_get_map_update_index = 0, -1, -100
        self.pose, self.cov = np.zeros(3, np.float32), np.zeros((3, 3), np.float32)

    def publish_map(self, stamp):
        """publishMap: the payload of level 0 (the grid's isFree / isOccupied), rebuilt when the update index moved."""
        lo, _ = self.proc.level(0)
        data = np.full(lo.shape, -1, np.int8)
        data[lo < 0] = 0
        data[lo > 0] = 100
        rebuilt = self.last_get_map_update_index != self.update_index
        self.last_get_map_update_index = self.update_index
        return dict(scan_index=self.scans, stamp=tuple(int(v) for v in stamp), info=dict(self.info), payload=data,
                    rebuilt=rebuilt)

    def process(self, ranges, stamps):
        amin, inc, rmin, rmax = self.geometry
        p = self.p
        out = dict(pose=[], pose_msg=[], cov=[], tf=[], map_updated=[], n_points=[], maps=[])
        for r, s in zip(np.asarray(ranges, np.float32), np.asarray(stamps, np.uint32)):
            tick = self.schedule.before(s)
            if tick is not None:
                out["maps"].append(self.publish_map(tick))
            pts = scans_port.project(r, amin, inc, rmin, rmax, 30.0)
            dc, origo = to_data_container(pts, self.mount, self.scale, p["laser_min_dist"], p["laser_max_dist"],
                                          p["use_max_scan_range"], p["laser_z_min_value"], p["laser_z_max_value"])
            self.pose, cov = self.proc.update(dc, origo, self.pose)  # startEstimate = getLastScanMatchPose()
            self.cov = cov
            if self.proc.map_updated:
                self.update_index += 1
            msg, c36, tf = pose_message(self.pose, self.cov)
            out["pose"].append(self.pose.copy())
            out["pose_msg"].append(msg)
            out["cov"].append(c36)
            out["tf"].append(tf)
            out["map_updated"].append(self.proc.map_updated)
            out["n_points"].append(len(dc))
            self.scans += 1
        for k in ("pose_msg", "cov", "tf"):
            out[k] = np.array(out[k], np.float64).reshape(-1, {"pose_msg": 7, "cov": 36, "tf": 7}[k])
        out["pose"] = np.array(out["pose"], np.float32).reshape(-1, 3)
        out["map_updated"] = np.array(out["map_updated"], bool)
        out["n_points"] = np.array(out["n_points"], np.int32)
        return out

    def close(self):
        self.proc.close()
