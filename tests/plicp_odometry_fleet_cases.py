"""Streams for the lesson3 odometry node fleet (b2s_plicp_odom_create_fleet / _process_fleet), built on
plicp_odometry_cases.py: range fields that change inside a recording, lasers of 3 to 2408 beams over 270 and 360 deg,
and mounts and parameter sets that differ between recordings.

A stream here carries its own laser (n_beams, angle_min, angle_increment as float32) and each scan's float32
(range_min, range_max).  The restatement of a stream is the C restatement orc_plicp_odometry on the scans NaN-masked
by their own fields with fields (-inf, inf), the CSM stand-in's own rule (oracle/shim/csm/csm_all.h): the node keeps
the valid flags each message's fields gave it, the key frame's included, and a reading is valid exactly when it is
inside its own message's fields.  The node's answers come from the unmodified node fed each message's own fields,
live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

import plicp_odometry_cases as pc

synth, abi, plicp = pc.synth, pc.abi, pc.plicp

RANGE = (0.1, 30.0)


def laser(n, fov_deg):
    """(n_beams, angle_min, angle_increment) of an n-beam laser over fov_deg, float32 fields: a 360 deg laser does not
    repeat its first beam."""
    fov = math.radians(fov_deg)
    inc = fov / n if fov_deg >= 360 else fov / (n - 1)
    return int(n), float(np.float32(-fov / 2)), float(np.float32(inc))


HOKUYO = (int(pc.LASER.n_readings), float(pc.FIELDS[0]), float(pc.FIELDS[1]))


def cast(world, base_pose, mount, las, rng, sigma):
    """pc.cast for a laser of its own: ranges of `las` on `mount` with the robot at base_pose."""
    qx, qy, qz, qw = mount[3:]
    xx, xy, zz = 1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qy * qy)
    c, s = math.cos(base_pose[2]), math.sin(base_pose[2])
    px = base_pose[0] + c * mount[0] - s * mount[1]
    py = base_pose[1] + s * mount[0] + c * mount[1]
    sign = 1 if zz > 0 else -1
    lz = synth.Laser(n_readings=las[0], min_angle=las[1] * sign, angular_resolution=las[2] * sign)
    return synth.cast_scan(world, (px, py, base_pose[2] + math.atan2(xy, xx)), lz, rng, sigma)


def stream(seed, steps, las=HOKUYO, mount=pc.IDENTITY, limits=None, params=None, sigma=0.005, dt=0.1):
    """steps [S][3] base motions as pc.stream; limits: {scan index: (range_min, range_max)} overriding RANGE."""
    rng = np.random.default_rng(seed)
    world = synth.make_world(seed)
    pose = np.zeros(3)
    ranges = []
    for k in range(len(steps) + 1):
        if k:
            f, l, t = steps[k - 1]
            c, s = math.cos(pose[2]), math.sin(pose[2])
            pose = pose + np.array([c * f - s * l, s * f + c * l, t])
        ranges.append(cast(world, pose, mount, las, rng, sigma))
    S = len(ranges)
    lim = np.tile(np.float32(RANGE), (S, 1))
    for k, v in (limits or {}).items():
        lim[k] = v
    t = 1000.0 + dt * np.arange(S)
    stamps = np.stack([np.floor(t), np.round((t - np.floor(t)) * 1e9)], 1).astype(np.uint32)
    return dict(ranges=np.array(ranges).astype(np.float32), stamps=stamps, mount=tuple(mount),
                params=dict(params or {}), laser=las, limits=lim)


def _streams():
    d = math.radians
    fwd = [(0.03, 0.0, d(0.3))] * 20
    slow = [(0.01, 0.0, d(0.2))] * 20
    every4 = dict(kf_scan_count=4, kf_dist_linear=0.5)
    off = (0.2, -0.1, 0.3) + pc.rpy_quaternion(0.0, 0.0, 0.3)
    return {
        # range_max dropped below some readings for a few scans
        "range_max_drop": stream(21, fwd, limits={k: (0.1, 4.0) for k in range(6, 10)}),
        # range_min raised above some readings for a few scans
        "range_min_raise": stream(22, fwd, limits={k: (4.0, 30.0) for k in range(8, 12)}),
        # the first key frame converted under a short range_max, the scans matched against it under the full one
        "keyframe_fields": stream(23, slow, limits={0: (0.1, 5.0)}, params=dict(kf_scan_count=6, kf_dist_linear=0.5)),
        # promotions every 4th scan (scan-count rule); the fields change on the scan right after the one at scan 4
        # and again after the one at scan 12
        "fields_after_promotion": stream(24, slow, params=every4,
                                         limits={**{k: (0.1, 6.0) for k in range(5, 13)},
                                                 **{k: (0.6, 30.0) for k in range(13, 21)}}),
        "laser_360_360": stream(25, fwd, las=laser(360, 360)),
        "laser_720_360": stream(26, fwd, las=laser(720, 360), limits={k: (0.1, 5.0) for k in range(4, 7)}),
        "laser_720_270": stream(27, fwd, las=laser(720, 270)),
        "laser_2048_360": stream(28, fwd[:12], las=laser(2048, 360)),
        "laser_2408_270": stream(29, fwd[:12], las=laser(2408, 270), limits={k: (0.3, 8.0) for k in range(5, 8)}),
        "laser_3": stream(30, fwd[:8], las=laser(3, 270)),
        "laser_4": stream(31, fwd[:8], las=laser(4, 360)),
        # mounts and parameter sets of their own
        "mount_launch_720": stream(32, [(0.03, 0.0, d(1.0))] * 16, las=laser(720, 360), mount=pc.LAUNCH_MOUNT,
                                   params=dict(kf_dist_angular=0.03, max_iterations=8, outliers_maxPerc=0.85)),
        "mount_offset_1440": stream(33, [(0.02, 0.01, d(-0.8))] * 16, las=laser(1440, 360), mount=off,
                                    params=dict(kf_dist_linear=0.06, kf_scan_count=5, max_correspondence_dist=0.5,
                                                max_linear_correction=0.4),
                                    limits={k: (0.2, 7.0) for k in range(9, 17)}),
    }


STREAMS = _streams()


def odom_params(st):
    return pc.odom_params(st)


def masked(st) -> np.ndarray:
    """Each scan's readings NaN where outside its own message's fields (r > range_min && r < range_max)."""
    r, lim = st["ranges"], st["limits"]
    keep = (r > lim[:, :1]) & (r < lim[:, 1:])
    return np.where(keep, r, np.float32(np.nan)).astype(np.float32)


def restate(st) -> np.ndarray:
    """orc_plicp_odometry on the masked scans with fields (-inf, inf) -> structured array of plicp.STEP_DTYPE."""
    from oracle import plicp_odometry_port
    n, amin, ainc = st["laser"]
    return plicp_odometry_port.odometry(odom_params(st), (amin, ainc, -np.inf, np.inf), masked(st), st["stamps"])


def restate_uniform(st) -> np.ndarray:
    """The existing orc_plicp_odometry over the stream's ranges with the scans' first fields for every scan."""
    from oracle import plicp_odometry_port
    n, amin, ainc = st["laser"]
    return plicp_odometry_port.odometry(odom_params(st), (amin, ainc, *st["limits"][0]), st["ranges"], st["stamps"])


def run_node(st) -> np.ndarray:
    """The unmodified node (oracle/ref_lesson3.cpp) over a stream, every LaserScan with its own range fields ->
    structured array [S] of plicp.STEP_DTYPE (reference_scan tracked from the keyframe flags, as ref_lesson3.run)."""
    from oracle import ref_lesson3
    L = ref_lesson3.lib()
    L.ref_plicp_clear_params()
    for k, v in st["params"].items():
        L.ref_plicp_param(k.encode(), float(v))
    m = np.ascontiguousarray(st["mount"], np.float64)
    L.ref_plicp_new(m.ctypes.data_as(C.POINTER(C.c_double)))
    n, amin, ainc = st["laser"]
    r = np.ascontiguousarray(st["ranges"], np.float32)
    out = np.zeros(len(r), plicp.STEP_DTYPE)
    kf = -1
    for s in range(len(r)):
        f = np.array([amin, ainc, *st["limits"][s]], np.float32)
        rc = L.ref_plicp_scan(int(st["stamps"][s][0]), int(st["stamps"][s][1]), f.ctypes.data_as(C.POINTER(C.c_float)),
                              n, r[s].ctypes.data_as(C.POINTER(C.c_float)), out[s:s + 1].ctypes.data)
        if rc != 0:
            raise RuntimeError("the lesson3 node threw (a CSM switch the stand-in refuses)")
        if out[s]["published"]:
            out[s]["reference_scan"] = kf
        if out[s]["keyframe"]:
            kf = s
    return out


def node_answers(live):
    """{stream name: pc.pack(node run)} from the unmodified node, live or replayed."""
    from reference_record import Recording
    rec = Recording("test_plicp_odometry_fleet_reference__node_streams", live)
    out = {}
    for name, st in STREAMS.items():
        out[name] = rec.value(name, lambda st=st: pc.pack(run_node(st)),
                              inputs=(st["ranges"], st["stamps"], st["limits"], list(st["laser"]), list(st["mount"]),
                                      sorted(st["params"].items())))
    rec.save()
    return out


def all_streams():
    """{name: stream} of every old stream (on the Hokuyo laser with constant fields) and every new one."""
    out = {}
    for name, st in pc.STREAMS.items():
        out[name] = dict(st, laser=HOKUYO, limits=np.tile(pc.FIELDS[2:4], (len(st["ranges"]), 1)).astype(np.float32))
    out.update(STREAMS)
    return out
