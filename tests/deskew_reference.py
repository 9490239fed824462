"""Independent float64 reference of lesson5's CorrectLaserScan (lidar_undistortion.cc:339-447), written from the node's
source and from the documented mathematics of pcl::getTransformation and Eigen's Affine3f, not from the restatement
(oracle/deskew_oracle.c) or the kernel (csrc/lidar_undistortion.cu).

For beam i of a scan:
  - angle_i = angle_min + i * angle_increment summed in float32, as CreateAngleCache sums the LaserScan's float fields
    with an unsigned index; cos / sin of it in float64.  p_i = (r_i cos, r_i sin, 1).
  - t_i = time_start + i * time_increment.
  - with use_imu, the rotation (roll, pitch, yaw) at t_i is ComputeRotation's: `front` is the first table entry below
    imu_last whose stamp is later than t_i (imu_last if none); past the stamp of `front`, or with front == 0, the entry
    itself; otherwise the linear interpolation between front - 1 and front.
  - with use_odom, the translation is odom_incre * (t_i - odom_start) / (odom_end - odom_start).
  - R = Rz(yaw) Ry(pitch) Rx(roll) (pcl::getTransformation), and the corrected point is R_0^T (R_i p_i + t_i - t_0),
    where 0 is the first valid beam of the scan (transStartInverse * transFinal).
  - a beam is valid when its range is finite and inside [range_min, range_max]; skipped beams are (0, 0, 0).
Everything after the beam angle is float64; the node and the kernel round the angles, the translation, every matrix
coefficient and every product to float32.

Bound (per component, returned by `deskew`): where the poses of beam i and of beam 0 are both exactly zero the float path is exact
up to the final rounding of the output, so |got - want| <= 2^-24 |want|.  Otherwise the float32 path makes these errors,
each at most 2^-24 relative per rounding:
  - the three rotation angles of each pose are rounded: a turn of 2^-24 |angle| each, moving a point by at most
    2^-24 (|theta_i|_1 + |theta_0|_1)(|p|_1 + |t_i|_1 + |t_0|_1);
  - every coefficient of getTransformation is at most four roundings (cos / sin, D*E, A*DF, the difference), the
    cofactor inverse adds about three more per coefficient (a 2x2 determinant, the product with 1/det), the product of
    the two transforms two more (a three-term sum), each on coefficients of magnitude <= 1; the matrix-vector sum in
    double then carries those coefficient errors times |p|_1, and the translations times their magnitude.
Taken together: |got - want| <= 2^-24 |want| + K 2^-24 (1 + |theta_i|_1 + |theta_0|_1)(|p|_1 + |t_i|_1 + |t_0|_1)
with K = 8, about the sum of the roundings counted above on one row.  A wrong composition order, swapped roll and
pitch, swapped interpolation weights or a start pose from the wrong beam all move points by the motion between two
poses (milliradians and millimetres and up), orders of magnitude above it."""
from __future__ import annotations

import numpy as np

EPS = 2.0 ** -24
K = 8.0


def _field(s, name):
    return s[name] if isinstance(s, dict) else getattr(s, name)


def rotation(roll, pitch, yaw):
    """R = Rz(yaw) Ry(pitch) Rx(roll) for arrays of angles -> [..., 3, 3]."""
    cx, sx, cy, sy, cz, sz = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    o, z = np.ones_like(cx), np.zeros_like(cx)
    rx = np.stack([np.stack([o, z, z], -1), np.stack([z, cx, -sx], -1), np.stack([z, sx, cx], -1)], -2)
    ry = np.stack([np.stack([cy, z, sy], -1), np.stack([z, o, z], -1), np.stack([-sy, z, cy], -1)], -2)
    rz = np.stack([np.stack([cz, -sz, z], -1), np.stack([sz, cz, z], -1), np.stack([z, z, o], -1)], -2)
    return rz @ ry @ rx


def beam_angles(n, angle_min, angle_increment):
    """CreateAngleCache: float32 angle, float64 cos / sin."""
    a = np.float32(angle_min) + np.arange(n, dtype=np.uint32).astype(np.float32) * np.float32(angle_increment)
    return a.astype(np.float64)


def poses(s, n, imu_time, rot_x, rot_y, rot_z):
    """(angles [n, 3] roll / pitch / yaw, translations [n, 3]) of every beam, float64."""
    t = _field(s, "time_start") + np.arange(n) * _field(s, "time_increment")
    ang, pos = np.zeros((n, 3)), np.zeros((n, 3))
    if _field(s, "use_imu"):
        last = int(_field(s, "imu_last"))
        T = np.asarray(imu_time, np.float64)[:last + 1]
        R = np.stack([np.asarray(a, np.float64)[:last + 1] for a in (rot_x, rot_y, rot_z)], -1)
        front = np.searchsorted(T[:last], t, side="right")  # first entry below imu_last stamped later than t
        hold = (t > T[front]) | (front == 0)
        back = np.maximum(front - 1, 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            span = T[front] - T[back]
            wf, wb = (t - T[back]) / span, (T[front] - t) / span
            lerp = R[front] * wf[:, None] + R[back] * wb[:, None]
        ang = np.where(hold[:, None], R[front], lerp)
    if _field(s, "use_odom"):
        ratio = (t - _field(s, "odom_start_time")) / (_field(s, "odom_end_time") - _field(s, "odom_start_time"))
        pos = np.asarray(_field(s, "odom_incre")[:], np.float64)[None, :] * ratio[:, None]
    return ang, pos


def valid(ranges, s):
    r = np.asarray(ranges, np.float32)
    return np.isfinite(r) & ~(r < np.float32(_field(s, "range_min"))) & ~(r > np.float32(_field(s, "range_max")))


def deskew(ranges, angle_min, angle_increment, s, imu_time, rot_x, rot_y, rot_z):
    """-> (corrected points [n, 3] float64, bound [n, 3]); skipped beams are 0 with a bound of 0."""
    r = np.asarray(ranges, np.float32)
    n = len(r)
    ok = valid(r, s)
    out, bnd = np.zeros((n, 3)), np.zeros((n, 3))
    if not ok.any():
        return out, bnd
    a = beam_angles(n, angle_min, angle_increment)
    rv = np.where(ok, r, 0).astype(np.float64)
    p = np.stack([rv * np.cos(a), rv * np.sin(a), np.ones(n)], -1)
    ang, pos = poses(s, n, imu_time, rot_x, rot_y, rot_z)
    f = int(np.argmax(ok))
    Ri, R0 = rotation(ang[:, 0], ang[:, 1], ang[:, 2]), rotation(*ang[f])
    world = np.einsum("nij,nj->ni", Ri, p) + pos - pos[f]
    q = world @ R0  # R_0^T applied to every row
    out[ok] = q[ok]
    moving = (np.abs(ang).sum(1) + np.abs(pos).sum(1) + np.abs(ang[f]).sum() + np.abs(pos[f]).sum()) > 0
    scale = (1 + np.abs(ang).sum(1) + np.abs(ang[f]).sum()) * (np.abs(p).sum(1) + np.abs(pos).sum(1) + np.abs(pos[f]).sum())
    b = EPS * np.abs(q) * (1 + 2.0 ** -20) + (moving * K * EPS * scale)[:, None]
    bnd[ok] = b[ok]
    return out, bnd


def check(got, ranges, angle_min, angle_increment, s, imu_time, rot_x, rot_y, rot_z):
    """Assert got [n, 3] float32 within the bound of the reference and zero on skipped beams; returns the largest
    ratio |got - want| / bound."""
    want, bnd = deskew(ranges, angle_min, angle_increment, s, imu_time, rot_x, rot_y, rot_z)
    ok = valid(ranges, s)
    got = np.asarray(got, np.float64)
    assert np.all(got[~ok] == 0), "a skipped beam is not (0, 0, 0)"
    err = np.abs(got - want)
    bad = err > bnd
    assert not bad.any(), (f"{bad.sum()} components outside the bound, first beam {np.argwhere(bad)[0][0]}: "
                           f"got {got[bad][:3]}, want {want[bad][:3]}, bound {bnd[bad][:3]}")
    return float((err[ok] / np.maximum(bnd[ok], 1e-300)).max()) if ok.any() else 0.0
