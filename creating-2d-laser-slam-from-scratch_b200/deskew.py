"""ctypes harness over the C ABI — lesson5 motion de-skew (LidarUndistortion, lidar_undistortion.cc): the batched
CorrectLaserScan on the device plus the per-scan host preparation (IMU angle integration, odometry increment)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .matcher import check, lib, f64, _d


class DeskewScan(C.Structure):
    """b2s_deskew_scan (include/b200slam.h)."""
    _fields_ = [("time_start", C.c_double), ("time_increment", C.c_double), ("range_min", C.c_float), ("range_max", C.c_float),
                ("use_imu", C.c_int32), ("use_odom", C.c_int32), ("imu_last", C.c_int32), ("reserved", C.c_int32),
                ("odom_start_time", C.c_double), ("odom_end_time", C.c_double), ("odom_incre", C.c_float * 3),
                ("reserved2", C.c_float)]


class ImuMsg(C.Structure):
    """b2s_imu_msg: header.stamp and angular_velocity of a sensor_msgs/Imu."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("angular_velocity", C.c_double * 3)]


class OdomMsg(C.Structure):
    """b2s_odom_msg: header.stamp, pose.pose.position and pose.pose.orientation (x, y, z, w) of a nav_msgs/Odometry."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("position", C.c_double * 3), ("orientation", C.c_double * 4)]


class NodeScan(C.Structure):
    """b2s_deskew_node_scan: one LaserScan's per-scan fields and the messages delivered before its callback."""
    _fields_ = [("sec", C.c_uint32), ("nsec", C.c_uint32), ("time_increment", C.c_float), ("range_min", C.c_float),
                ("range_max", C.c_float), ("imu_arrived", C.c_int32), ("odom_arrived", C.c_int32),
                ("reserved", C.c_int32)]


class DeskewLaser(C.Structure):
    """b2s_deskew_laser: what a node of DeskewNodeBatch takes from its first scan."""
    _fields_ = [("angle_min", C.c_float), ("angle_increment", C.c_float), ("n_beams", C.c_int32), ("use_imu", C.c_int32),
                ("use_odom", C.c_int32), ("reserved", C.c_int32)]


# numpy record layouts of the structs, for whole logs
IMU_DTYPE, ODOM_DTYPE, SCAN_DTYPE, STATE_DTYPE = (np.dtype(s) for s in (ImuMsg, OdomMsg, NodeScan, DeskewScan))
# B2S_DESKEW_* (include/b200slam.h); CACHED only in DeskewNodeBatch rows
PUBLISHED, HELD, WAIT_IMU, IMU_EMPTY, WAIT_ODOM, ODOM_EMPTY, UNDEFINED, CACHED = range(8)


def imu_log(stamps, angular_velocity):
    """stamps [N, 2] (sec, nsec), angular_velocity [N, 3] -> IMU_DTYPE [N]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), IMU_DTYPE)
    a["sec"], a["nsec"], a["angular_velocity"] = st[:, 0], st[:, 1], np.asarray(angular_velocity, np.float64).reshape(-1, 3)
    return a


def odom_log(stamps, position, orientation):
    """stamps [N, 2], position [N, 3], orientation [N, 4] (x, y, z, w) -> ODOM_DTYPE [N]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), ODOM_DTYPE)
    a["sec"], a["nsec"] = st[:, 0], st[:, 1]
    a["position"], a["orientation"] = np.asarray(position).reshape(-1, 3), np.asarray(orientation).reshape(-1, 4)
    return a


def node_scans(stamps, time_increment, range_min, range_max, imu_arrived, odom_arrived):
    """per-scan stamps [S, 2] (sec, nsec), float fields (scalars or [S]) and arrival counts [S] -> SCAN_DTYPE [S]"""
    st = np.asarray(stamps, np.uint32).reshape(-1, 2)
    a = np.zeros(len(st), SCAN_DTYPE)
    a["sec"], a["nsec"] = st[:, 0], st[:, 1]
    a["time_increment"], a["range_min"], a["range_max"] = time_increment, range_min, range_max
    a["imu_arrived"], a["odom_arrived"] = imu_arrived, odom_arrived
    return a


_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
        L.b2s_deskew_integrate_imu.argtypes = [C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, dp, dp, dp, dp]
        L.b2s_deskew_integrate_imu.restype = C.c_int32
        L.b2s_deskew_odom_increment.argtypes = [dp, dp, fp]
        L.b2s_deskew_odom_increment.restype = None
        L.b2s_lidar_undistort.argtypes = [C.c_int, C.c_int, fp, C.c_double, C.c_double, C.POINTER(DeskewScan), dp, dp, dp, dp,
                                          C.c_int, fp, C.c_int, C.c_void_p]
        vp = C.c_void_p
        L.b2s_lidar_undistortion_node.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, vp, vp, C.c_int,
                                                  vp, C.c_int, vp, vp, vp, vp, C.c_int, vp]
        L.b2s_deskew_node_create.argtypes = [C.c_int, C.POINTER(DeskewLaser), C.c_int, vp, C.POINTER(vp)]
        L.b2s_deskew_node_destroy.argtypes = [vp]
        L.b2s_deskew_node_destroy.restype = None
        L.b2s_deskew_node_reset.argtypes = [vp, C.c_int]
        L.b2s_deskew_node_process.argtypes = [vp] * 11
        _bound = True
    return L


def integrate_imu(stamps, angular_velocity, scan_start, scan_end, capacity=2000, fn=None):
    """PruneImuDeque's integration -> (imu_last, imu_time, rot_x, rot_y, rot_z)."""
    fn = fn or _bind().b2s_deskew_integrate_imu
    st, av = f64(stamps), f64(angular_velocity).reshape(-1, 3)
    t, x, y, z = (np.zeros(capacity) for _ in range(4))
    last = fn(len(st), _d(st), _d(av), float(scan_start), float(scan_end), capacity, _d(t), _d(x), _d(y), _d(z))
    return int(last), t, x, y, z


def odom_increment(start_pose, end_pose, fn=None):
    fn = fn or _bind().b2s_deskew_odom_increment
    out = np.zeros(3, np.float32)
    fn(_d(f64(start_pose)), _d(f64(end_pose)), out.ctypes.data_as(C.POINTER(C.c_float)))
    return out


def undistort(ranges, angle_min, angle_increment, scans, imu_time, rot_x, rot_y, rot_z, device=0, stream=None):
    """ranges [B, n] float32, scans: list of DeskewScan, IMU tables [B, stride] -> corrected cloud [B, n, 3] float32."""
    L = _bind()
    r = np.ascontiguousarray(ranges, np.float32)
    B, n = r.shape
    arr = (DeskewScan * B)(*scans)
    t, x, y, z = (np.ascontiguousarray(a, np.float64).reshape(B, -1) for a in (imu_time, rot_x, rot_y, rot_z))
    out = np.zeros((B, n, 3), np.float32)
    fp = C.POINTER(C.c_float)
    check(L.b2s_lidar_undistort(B, n, r.ctypes.data_as(fp), float(angle_min), float(angle_increment), arr, _d(t), _d(x), _d(y),
                                _d(z), t.shape[1], out.ctypes.data_as(fp), device, C.c_void_p(stream) if stream else None))
    return out


def undistort_recording(use_imu, use_odom, angle_min, angle_increment, scans, ranges, imu=(), odom=(), device=0,
                        stream=None, out=None):
    """The whole node over one recording (b2s_lidar_undistortion_node).  scans: SCAN_DTYPE [S] (node_scans), ranges
    [S, n] float32, imu / odom: IMU_DTYPE / ODOM_DTYPE logs in delivery order.  out: an optional float32 [S, n, 3]
    array for the clouds (page-locked memory speeds the copy).  -> (status [S] int32, state [S] STATE_DTYPE,
    xyz [S, n, 3] float32): rows are indexed by the corrected scan."""
    L = _bind()
    r = np.ascontiguousarray(ranges, np.float32)
    S, n = r.shape
    sc = np.ascontiguousarray(scans, SCAN_DTYPE)
    im, od = np.ascontiguousarray(imu, IMU_DTYPE), np.ascontiguousarray(odom, ODOM_DTYPE)
    assert len(sc) == S
    status, state = np.zeros(S, np.int32), np.zeros(S, STATE_DTYPE)
    xyz = np.zeros((S, n, 3), np.float32) if out is None else out
    assert xyz.dtype == np.float32 and xyz.shape == (S, n, 3) and xyz.flags.c_contiguous
    check(L.b2s_lidar_undistortion_node(int(use_imu), int(use_odom), float(angle_min), float(angle_increment), n, S,
                                        sc.ctypes.data, r.ctypes.data, len(im), im.ctypes.data, len(od), od.ctypes.data,
                                        status.ctypes.data,
                                        state.ctypes.data, xyz.ctypes.data, device, stream))
    return status, state, xyz


class DeskewNodeBatch:
    """B lesson5 LidarUndistortion nodes on the device (b2s_deskew_node_*), one laser per recording, fed in parts: the
    handle keeps every node's held scan, queues and odometry messages between calls.  lasers: a sequence of
    DeskewLaser."""

    def __init__(self, lasers, device=0, stream=None):
        L = _bind()
        self.lasers = (DeskewLaser * len(lasers))(*lasers)
        self.batch = len(lasers)
        self.n = np.array([l.n_beams for l in lasers], np.int32)
        self._h = C.c_void_p()
        check(L.b2s_deskew_node_create(self.batch, self.lasers, device, C.c_void_p(stream) if stream else None,
                                       C.byref(self._h)))

    def process(self, chunks):
        """chunks: one (scans, ranges, imu, odom) per recording, or None for nothing: scans SCAN_DTYPE [S] with arrival
        counts into this chunk's imu / odom (IMU_DTYPE / ODOM_DTYPE logs), ranges [S, n_beams] float32.  -> one
        (status [S] int32, state [S] STATE_DTYPE, xyz [S, n_beams, 3] float32) per recording: rows are
        callback-indexed, row k what the callback of the chunk's k-th scan did (CACHED for the node's first scan)."""
        if len(chunks) != self.batch:
            raise ValueError("one chunk (or None) per recording of the handle")
        sc, rg, im, od = [], [], [], []
        for b, c in enumerate(chunks):
            s, r, i, o = c if c is not None else (np.zeros(0, SCAN_DTYPE), np.zeros((0, self.n[b]), np.float32),
                                                  np.zeros(0, IMU_DTYPE), np.zeros(0, ODOM_DTYPE))
            s, r = np.asarray(s, SCAN_DTYPE).reshape(-1), np.asarray(r, np.float32)
            if r.size != len(s) * self.n[b]:
                raise ValueError(f"recording {b}: ranges are [n_scans, {self.n[b]}]")
            sc.append(s), rg.append(r.reshape(-1)), im.append(np.asarray(i, IMU_DTYPE).reshape(-1))
            od.append(np.asarray(o, ODOM_DTYPE).reshape(-1))
        counts = [np.array([len(a) for a in x], np.int32) for x in (sc, im, od)]
        S, R, I, O = (np.ascontiguousarray(np.concatenate(x)) for x in (sc, rg, im, od))
        total = len(S)
        status, state = np.zeros(total, np.int32), np.zeros(total, STATE_DTYPE)
        xyz = np.zeros(len(R) * 3, np.float32)
        check(_bind().b2s_deskew_node_process(self._h, counts[0].ctypes.data, S.ctypes.data, R.ctypes.data,
                                              counts[1].ctypes.data, I.ctypes.data, counts[2].ctypes.data,
                                              O.ctypes.data, status.ctypes.data, state.ctypes.data, xyz.ctypes.data))
        out, q, f = [], 0, 0
        for b, k in enumerate(counts[0]):
            k, m = int(k), int(k) * int(self.n[b]) * 3
            out.append((status[q:q + k], state[q:q + k], xyz[f:f + m].reshape(k, int(self.n[b]), 3)))
            q, f = q + k, f + m
        return out

    def reset(self, recording=-1):
        check(_bind().b2s_deskew_node_reset(self._h, int(recording)))

    def close(self):
        if self._h:
            _bind().b2s_deskew_node_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def laser_of(rec, flags):
    """The DeskewLaser of a recording dict (amin, ainc, ranges [S, n]) fed with flags (use_imu, use_odom)."""
    return DeskewLaser(float(rec["amin"]), float(rec["ainc"]), int(np.shape(rec["ranges"])[1]), int(flags[0]),
                       int(flags[1]), 0)


def split_recording(rec, cuts, imu_splits=None, odom_splits=None):
    """Cut one recording into consecutive chunks for DeskewNodeBatch.process.  rec: a dict with scans (SCAN_DTYPE,
    arrival counts into the whole logs), ranges [S, n], imu and odom (whole logs).  cuts: non-decreasing scan indices
    in [0, S]; chunk c holds scans [cuts[c - 1], cuts[c]) (cuts[-1] = 0) and the last chunk the rest, so a repeated
    cut gives a chunk without scans.  imu_splits / odom_splits [len(cuts)]: the message index where chunk c's
    messages end, anywhere from the arrival count of the scan before cuts[c] to that of scan cuts[c] (default: the
    former, every later message goes with the next chunk).  The last chunk takes every remaining message.  Arrival
    counts are rebased to each chunk's own messages.  -> list of (scans, ranges, imu, odom)."""
    sc, S = rec["scans"], len(rec["scans"])
    cuts = [int(c) for c in cuts]
    if any(not 0 <= c <= S for c in cuts) or any(b < a for a, b in zip(cuts, cuts[1:])):
        raise ValueError("cuts are non-decreasing scan indices in [0, S]")

    def splits(given, field, log_len):
        lo = [int(sc[field][c - 1]) if c > 0 else 0 for c in cuts]
        hi = [int(sc[field][c]) if c < S else log_len for c in cuts]
        m = lo if given is None else [int(x) for x in given]
        if len(m) != len(cuts) or any(not a <= x <= b for a, x, b in zip(lo, m, hi)) or any(y < x for x, y in zip(m, m[1:])):
            raise ValueError(f"{field} splits do not decrease and lie between the arrival counts around each cut")
        return [0] + m + [log_len]

    mi = splits(imu_splits, "imu_arrived", len(rec["imu"]))
    mo = splits(odom_splits, "odom_arrived", len(rec["odom"]))
    edges = [0] + cuts + [S]
    out = []
    for c in range(len(edges) - 1):
        s = sc[edges[c]:edges[c + 1]].copy()
        s["imu_arrived"] -= mi[c]
        s["odom_arrived"] -= mo[c]
        out.append((s, rec["ranges"][edges[c]:edges[c + 1]], rec["imu"][mi[c]:mi[c + 1]], rec["odom"][mo[c]:mo[c + 1]]))
    return out
