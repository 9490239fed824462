"""Restatement of lesson4's LaserScan -> DataContainer conversion (HectorMappingRos::scanCallback,
lesson4/src/hector_mapping/hector_slam.cc:186-205), written independently of the library:

  projectLaser(scan, cloud, range_cutoff)   laser_geometry's LaserProjection, sensor_msgs::PointCloud form (the package
                                            is not in the reference tree: restated from its published behaviour)
  rosPointCloudToDataContainer              hector_slam.cc:320-362

Double arithmetic is Python's float (IEEE binary64), transcendental functions are math.cos / math.sin (the C library's),
and every float32 step is a numpy float32 scalar operation, so each result is rounded where the C++ rounds it."""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32


def unit_vectors(angle_min, angle_increment, n):
    """getUnitVectors_: cos / sin(angle_min + (double)i * angle_increment), the float32 message fields widened."""
    a0, inc = float(f32(angle_min)), float(f32(angle_increment))
    out = []
    for i in range(n):
        a = a0 + float(i) * inc
        out.append((math.cos(a), math.sin(a)))
    return out


def project(ranges, angle_min, angle_increment, range_min, range_max, range_cutoff=30.0):
    """Laser-frame points [k, 3] float32 of the beams projectLaser keeps: range < cutoff (double; a negative cutoff
    means range_max) and range >= range_min (float)."""
    cutoff = float(f32(range_max)) if range_cutoff < 0 else float(range_cutoff)
    rmin = f32(range_min)
    r = np.asarray(ranges, np.float32).reshape(-1)
    pts = []
    for v, (ux, uy) in zip(r, unit_vectors(angle_min, angle_increment, len(r))):
        if float(v) < cutoff and v >= rmin:
            pts.append((f32(float(v) * ux), f32(float(v) * uy), f32(0.0)))
    return np.array(pts, np.float32).reshape(-1, 3)


def to_data_container(pts_xyz, laser_in_base=(0, 0, 0, 0), scale_to_map=20.0, min_dist=0.2, max_dist=30.0,
                      use_max_scan_range=20.0, z_min=-1.0, z_max=1.0):
    """rosPointCloudToDataContainer: DataContainer entries [k, 2] float32 (map-cell units) and origo [2]."""
    lb = [f32(v) for v in laser_in_base]
    lx, ly, lz = float(lb[0]), float(lb[1]), float(lb[2])
    c, s = math.cos(float(lb[3])), math.sin(float(lb[3]))
    scale = f32(scale_to_map)
    sqr_min, sqr_max = f32(min_dist) * f32(min_dist), f32(max_dist) * f32(max_dist)
    use = float(use_max_scan_range)
    zmin, zmax = f32(z_min), f32(z_max)
    out = []
    with np.errstate(all="ignore"):  # huge ranges square to inf in float32, as in the node
        for x, y, z in np.asarray(pts_xyz, np.float32).reshape(-1, 3):
            d = x * x + y * y
            if not (d > sqr_min and d < sqr_max):
                continue
            if x < f32(0.0) and d < f32(0.5):
                continue
            if float(d) > use * use:
                continue
            # laserTransform * Vector3(x, y, z) in tf's order, on the basis rows (c, -s, -0.0), (s, c, -0.0), (0, 0, 1)
            # that the library builds from the yaw: -0.0, not +0.0, in the third column
            xd, yd, zd = float(x), float(y), float(z)
            bx = (xd * c + yd * -s + zd * -0.0) + lx
            by = (xd * s + yd * c + zd * -0.0) + ly
            zl = f32(((xd * 0.0 + yd * 0.0 + zd * 1.0) + lz) - lz)
            if zl > zmin and zl < zmax:
                out.append((f32(bx) * scale, f32(by) * scale))
        origo = np.array([f32(lx) * scale, f32(ly) * scale], np.float32)
    return np.array(out, np.float32).reshape(-1, 2), origo


def scans(ranges, angle_min, angle_increment, range_min, range_max, range_cutoff=30.0, scale_to_map=20.0, **filt):
    """Both stages over [n_scans, n_ranges] ranges: ([per-scan DataContainer [k, 2]], origo [2])."""
    r = np.asarray(ranges, np.float32)
    if r.ndim != 2:
        r = r.reshape(1, -1)
    out, origo = [], None
    for row in r:
        pts = project(row, angle_min, angle_increment, range_min, range_max, range_cutoff)
        dc, origo = to_data_container(pts, scale_to_map=scale_to_map, **filt)
        out.append(dc)
    if origo is None:
        origo = to_data_container(np.zeros((0, 3), np.float32), scale_to_map=scale_to_map, **filt)[1]
    return out, origo
