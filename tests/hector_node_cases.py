"""Recordings for lesson4's Hector SLAM node (b2s_hector_node_*, oracle/hector_node_port.py): LaserScan ranges, stamps,
the node's parameters and the laser mount."""
from __future__ import annotations

import importlib
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
PKG = "creating-2d-laser-slam-from-scratch_b200"
synth = importlib.import_module(PKG + ".synth")
hector_node = importlib.import_module(PKG + ".hector_node")

f32 = np.float32
LASER = synth.Laser()
# beam 0 points along +x so that a range of 0.2f lands on the squared-threshold boundary exactly
GEOMETRY = (f32(LASER.min_angle), f32(LASER.angular_resolution), f32(0.1), f32(30.0))
BOUNDARY_GEOMETRY = (f32(0.0), f32(LASER.angular_resolution), f32(0.1), f32(30.0))
SMALL = dict(map_size=512)  # 25.6 m square: the walks stay inside it


def quat_rpy(roll, pitch, yaw):
    """Quaternion::setRPY in double (x, y, z, w)."""
    hy, hp, hr = yaw * 0.5, pitch * 0.5, roll * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


def mount(x=0.0, y=0.0, z=0.0, roll=0.0, pitch=0.0, yaw=0.0):
    return (x, y, z) + quat_rpy(roll, pitch, yaw)


def stamps_at(t0_sec, t0_nsec, dt_ns, n, gaps=()):
    """[n, 2] (sec, nsec): every dt_ns, with extra nanoseconds added from the given scan on (gaps = ((scan, ns), ...))."""
    t = t0_sec * 1_000_000_000 + t0_nsec
    out = []
    for i in range(n):
        for at, extra in gaps:
            if i == at:
                t += extra
        out.append((t // 1_000_000_000, t % 1_000_000_000))
        t += dt_ns
    return np.array(out, np.uint32)


def walk(seed, n, step_xy=0.05, step_th_deg=2.0, laser=LASER, room=(8.0, 6.0)):
    _, _, ranges = synth.make_trajectory(seed, n, laser, room[0], room[1], step_xy=step_xy, step_th_deg=step_th_deg)
    return ranges.astype(np.float32)


def laser(beams, angle_min, angle_increment, range_min=0.1, range_max=30.0):
    """A synth laser of `beams` beams from angle_min (radians, float32 message fields) and its LaserScan geometry."""
    amin, inc = f32(angle_min), f32(angle_increment)
    las = synth.Laser(n_readings=beams, min_angle=float(amin), max_angle=float(amin) + float(inc) * (beams - 1),
                      angular_resolution=float(inc), min_range=range_min, max_range=range_max)
    return las, (amin, inc, f32(range_min), f32(range_max))


RING, RING_GEOMETRY = laser(360, -math.pi, 2 * math.pi / 360, 0.15, 12.0)
DENSE, DENSE_GEOMETRY = laser(4096, -math.pi, 2 * math.pi / 4096, 0.1, 20.0)
# the Hokuyo swept from +135 deg down: beam 0 on the left, a negative angle_increment
CLOCKWISE, CLOCKWISE_GEOMETRY = laser(1081, -LASER.min_angle, -LASER.angular_resolution)
BIG_ROOM = (14.0, 10.0)  # walls up to about 17 m from the walk
FRONT = slice(520, 561)  # Hokuyo beams within 5 deg of straight ahead: x > 0, so the behind-the-robot rule keeps them


def _band(seed, n, lo, hi, beams=FRONT, r=None, exact=()):
    """A walk with the beams `beams` of every scan drawn from [lo, hi) (float32), and the values `exact` on the first
    of them."""
    r = walk(seed, n) if r is None else r
    rng = np.random.default_rng(seed)
    k = r[:, beams].shape[1]
    r[:, beams] = rng.uniform(lo, hi, (len(r), k)).astype(np.float32)
    np.clip(r[:, beams], f32(lo), np.nextafter(f32(hi), f32(0)), out=r[:, beams])
    for j, v in enumerate(exact):
        r[:, beams.start + j] = f32(v)
    return r


def _fields_lo(seed, n):
    """range_min 0.05: readings in [0.05, 0.1) that the 0.1 of the other cases would drop, and [0.03, 0.05) below it."""
    r = _band(seed, n, 0.05, 0.1, exact=(0.05, np.nextafter(f32(0.05), f32(0))))
    return _band(seed + 1, n, 0.03, 0.05, beams=slice(561, 566), r=r)


def _fields_40(seed, n):
    """range_max 40: readings in [30, 40) (30 itself among them) that projectLaser's 30 m cutoff drops, and (20, 30)
    that it keeps."""
    r = _band(seed, n, 30.0, 40.0, exact=(30.0, np.nextafter(f32(30.0), f32(0))))
    return _band(seed + 1, n, 20.0, 30.0, beams=slice(300, 330), r=r)


def _bad(seed, n):
    r = walk(seed, n)
    rng = np.random.default_rng(seed)
    bad = rng.random(r.shape) < 0.15
    r[bad] = rng.choice(np.array([np.nan, np.inf, -np.inf, 31.0, 45.0, 0.05], np.float32), int(bad.sum()))
    # points behind the robot within 0.5 m^2 (beams near +-180 deg at 0.5 m) and just outside it
    r[:, :20] = f32(0.5)
    r[:, -20:] = f32(0.75)
    return r


def _empty(seed, n, at):
    r = walk(seed, n)
    for i in at:
        r[i] = np.nan
    return r


def _boundary(seed, n):
    r = walk(seed, n)
    r[:, 0] = f32(0.2)   # x = 0.2f, y = 0: 0.2f * 0.2f = 0.040000003 > (float)(0.2 * 0.2) = 0.04: the node keeps it
    r[:, 1] = f32(0.2)
    return r


def cases():
    """name -> dict(params (ROS dict), mount, geometry, ranges, stamps)."""
    at40 = 25_000_000
    shipped = dict(hector_node.SHIPPED_LAUNCH)
    return {
        "defaults": dict(params={}, mount=mount(), geometry=GEOMETRY, ranges=walk(1, 12),
                         stamps=stamps_at(100, 0, 250_000_000, 12)),
        "shipped_launch": dict(params=shipped, mount=hector_node.SHIPPED_MOUNT, geometry=GEOMETRY, ranges=walk(2, 12),
                               stamps=stamps_at(200, 500_000_000, 250_000_000, 12)),
        "yaw_pi": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(0.0, 0.0, 0.254, yaw=3.1415926),
                       geometry=GEOMETRY, ranges=walk(11, 8), stamps=stamps_at(5, 0, at40, 8)),
        "upside_down": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(0.1, -0.05, 0.3, roll=math.pi),
                            geometry=GEOMETRY, ranges=walk(3, 10), stamps=stamps_at(5, 0, at40, 10)),
        "pitched_z_window": dict(params=dict(SMALL, laser_z_min_value=-0.3, laser_z_max_value=0.3, map_pub_period=0.1),
                                 mount=mount(0.05, 0.0, 0.4, pitch=0.12, yaw=0.3), geometry=GEOMETRY,
                                 ranges=walk(4, 10), stamps=stamps_at(5, 0, at40, 10)),
        "boundary_0.04f": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(), geometry=BOUNDARY_GEOMETRY,
                               ranges=_boundary(5, 8), stamps=stamps_at(7, 0, at40, 8)),
        "bad_ranges": dict(params=dict(SMALL, map_pub_period=0.05), mount=mount(0.12, 0.0, 0.2, yaw=0.05),
                           geometry=GEOMETRY, ranges=_bad(6, 10), stamps=stamps_at(9, 990_000_000, at40, 10)),
        "empty_scans": dict(params=dict(SMALL, map_pub_period=0.05), mount=mount(), geometry=GEOMETRY,
                            ranges=_empty(7, 10, (0, 1, 5, 6)), stamps=stamps_at(3, 0, at40, 10)),
        "rare_gate": dict(params=dict(SMALL, map_update_distance_thresh=50.0, map_update_angle_thresh=50.0,
                                      map_pub_period=0.05), mount=mount(), geometry=GEOMETRY, ranges=walk(8, 10),
                          stamps=stamps_at(3, 0, at40, 10)),
        "schedule_gaps": dict(params=dict(SMALL, map_pub_period=0.3), mount=mount(), geometry=GEOMETRY,
                              ranges=walk(9, 14),
                              # tick 0 = 10.9 s; a 5 s gap before scan 4 (16.0 s, exactly tick 17, across a
                              # second carry) publishes once, stamped with tick 1, then the next tick is 16.3 s
                              stamps=stamps_at(10, 900_000_000, 25_000_000, 14, gaps=((4, 5_000_000_000),))),
        "short_period": dict(params=dict(SMALL, map_pub_period=0.01), mount=mount(), geometry=GEOMETRY,
                             ranges=walk(10, 8), stamps=stamps_at(1, 0, at40, 8)),
        # ---- per-node map settings: each differs from every case above in the field it is named for ----
        "start_asym": dict(params=dict(SMALL, map_start_x=0.3, map_start_y=0.7, map_pub_period=0.1,
                                         map_update_distance_thresh=0.1, map_update_angle_thresh=0.1), mount=mount(),
                           geometry=GEOMETRY, ranges=walk(12, 12, step_xy=0.3), stamps=stamps_at(4, 0, at40, 12)),
        "start_asym_2": dict(params=dict(SMALL, map_start_x=0.65, map_start_y=0.35, map_pub_period=0.1,
                                           map_update_distance_thresh=0.1, map_update_angle_thresh=0.1),
                             mount=mount(0.08, 0.03, 0.2, yaw=-0.2), geometry=GEOMETRY,
                             ranges=walk(30, 12, step_xy=0.3), stamps=stamps_at(4, 0, at40, 12)),
        "res_0.1_levels_1": dict(params=dict(map_size=256, map_resolution=0.1, map_multi_res_levels=1,
                                             map_pub_period=0.1), mount=mount(), geometry=GEOMETRY,
                                 ranges=walk(14, 10), stamps=stamps_at(6, 0, at40, 10)),
        "res_0.025_levels_4": dict(params=dict(map_size=512, map_resolution=0.025, map_multi_res_levels=4,
                                               map_pub_period=0.1), mount=mount(), geometry=GEOMETRY,
                                   ranges=walk(15, 10), stamps=stamps_at(6, 0, at40, 10)),
        # 515 -> 257 -> 128 -> 64: the coarse levels drop a cell
        "res_0.075_odd_size": dict(params=dict(map_size=515, map_resolution=0.075, map_multi_res_levels=4,
                                               map_start_x=0.45, map_pub_period=0.1), mount=mount(),
                                   geometry=GEOMETRY, ranges=walk(16, 10), stamps=stamps_at(6, 0, at40, 10)),
        "factors": dict(params=dict(SMALL, update_factor_free=0.35, update_factor_occupied=0.7, map_pub_period=0.1),
                        mount=mount(), geometry=GEOMETRY, ranges=walk(17, 10), stamps=stamps_at(6, 0, at40, 10)),
        # ---- per-node lasers ----
        "ring_360": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(), geometry=RING_GEOMETRY,
                         ranges=walk(18, 10, laser=RING), stamps=stamps_at(8, 0, at40, 10)),
        "clockwise": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(0.05, 0.0, 0.1, yaw=0.4),
                          geometry=CLOCKWISE_GEOMETRY, ranges=walk(19, 10, laser=CLOCKWISE),
                          stamps=stamps_at(8, 0, at40, 10)),
        "dense_4096": dict(params=dict(SMALL, map_pub_period=0.1), mount=mount(), geometry=DENSE_GEOMETRY,
                           ranges=walk(20, 6, laser=DENSE), stamps=stamps_at(8, 0, at40, 6)),
        "fields_lo": dict(params=dict(SMALL, laser_min_dist=0.03, map_pub_period=0.1), mount=mount(),
                          geometry=GEOMETRY[:2] + (f32(0.05), GEOMETRY[3]), ranges=_fields_lo(21, 10),
                          stamps=stamps_at(8, 0, at40, 10)),
        "min_dist_0.5": dict(params=dict(SMALL, laser_min_dist=0.5, map_pub_period=0.1), mount=mount(),
                             geometry=GEOMETRY, ranges=_band(23, 10, 0.1, 0.5), stamps=stamps_at(8, 0, at40, 10)),
        # range_max 10 in the message: projectLaser is asked for 30 m, so the walls past 10 m stay
        "fields_hi": dict(params=dict(SMALL, use_max_scan_range=25.0, map_pub_period=0.1), mount=mount(),
                          geometry=GEOMETRY[:3] + (f32(10.0),), ranges=walk(24, 10, laser=LASER, room=BIG_ROOM),
                          stamps=stamps_at(8, 0, at40, 10)),
        "fields_40": dict(params=dict(SMALL, use_max_scan_range=50.0, laser_max_dist=50.0, map_pub_period=0.1),
                          mount=mount(), geometry=GEOMETRY[:3] + (f32(40.0),), ranges=_fields_40(25, 10),
                          stamps=stamps_at(8, 0, at40, 10)),
        "max_dist_8": dict(params=dict(SMALL, laser_max_dist=8.0, use_max_scan_range=12.0, map_pub_period=0.1),
                           mount=mount(), geometry=GEOMETRY, ranges=walk(27, 10, room=BIG_ROOM),
                           stamps=stamps_at(8, 0, at40, 10)),
        "use_range_5": dict(params=dict(SMALL, use_max_scan_range=5.0, map_pub_period=0.1), mount=mount(),
                            geometry=GEOMETRY, ranges=walk(28, 10), stamps=stamps_at(8, 0, at40, 10)),
        # a new laser through the pitched mount's z window
        "ring_pitched": dict(params=dict(SMALL, laser_z_min_value=-0.3, laser_z_max_value=0.3, map_pub_period=0.1),
                             mount=mount(0.05, 0.0, 0.4, pitch=0.12, yaw=0.3), geometry=RING_GEOMETRY,
                             ranges=walk(29, 10, laser=RING), stamps=stamps_at(8, 0, at40, 10)),
    }


def exact_tick_stamps():
    """Stamps where the tick 0 + 1 period (0.3 s from 10.9 s) is exactly a scan's stamp (11 s + 200 ms)."""
    return np.array([(10, 900_000_000), (11, 100_000_000), (11, 200_000_000), (11, 250_000_000)], np.uint32)


def uninitialised_rows(n_points):
    """Scans before the first that kept a beam: the node reports an uninitialised lastScanMatchCov there."""
    n = np.asarray(n_points)
    first = int(np.argmax(n > 0)) if (n > 0).any() else len(n)
    return np.arange(len(n)) < first
