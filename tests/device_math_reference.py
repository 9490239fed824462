"""mpmath references for the library functions that call libm: ros_math.cuh's quat_set_rpy, tf_get_rpy, tf_get_yaw and
tf2_get_yaw, and common.cuh's sensor_pose_of, on the records tests/device_math_check.cu writes (libm_records.bin:
float64 rows of [op, in[0..8], device out[0..3], host out[0..3]]).

The reference keeps every arithmetic operation of the C code in float64 (numpy scalars: IEEE, no contraction) and takes
each libm call correctly rounded from mpmath at 60 digits.  So the distance of a result from it comes from the libm calls
alone.  Each bound below composes the CUDA Math API's documented maxima (sin, cos, atan2, asin: 2 ulp), plus the half ulp
of the correctly rounded reference, through the formula:
- set_rpy: each component is a difference of two triple products of sines / cosines (|.| <= 1).  Three factors at
  2.5 ulp, the two product roundings and the final subtraction give <= 20 * 2^-53: 10 units of ulp(1.0).
- tf2_get_yaw, and tf_get_rpy's pitch and its singular branch: one atan2 or asin of the same double arguments: 2.5,
  bound 3 ulps of the result.
- tf_get_rpy's regular roll / yaw and tf_get_yaw: atan2(y / c, x / c) with c = cos(-asin(m20)); c only scales both
  arguments, but the two divisions re-round (<= 1 ulp on the ratio): 2.5 + 2, bound 6 ulps of the result.
- sensor_pose_of: x, y = robot + R(theta) offset: cos / sin at 2.5 ulp scaled by the offset, plus re-rounded products
  and sums: bound 4 units of ulp(max(|result|, |ox| + |oy|)).  The heading is arithmetic only: bound 0.
"""
import math

import mpmath
import numpy as np

OP_SET_RPY, OP_GET_RPY, OP_TF_GET_YAW, OP_TF2_GET_YAW, OP_SENSOR_POSE = 6, 7, 8, 9, 17
NAMES = {OP_SET_RPY: "set_rpy", OP_GET_RPY: "get_rpy", OP_TF_GET_YAW: "tf_get_yaw", OP_TF2_GET_YAW: "tf2_get_yaw",
         OP_SENSOR_POSE: "sensor_pose_of"}
N_OUT = {OP_SET_RPY: 4, OP_GET_RPY: 3, OP_TF_GET_YAW: 1, OP_TF2_GET_YAW: 1, OP_SENSOR_POSE: 3}
BOUND = {"set_rpy": 10.0, "get_rpy": 6.0, "tf_get_yaw": 6.0, "tf2_get_yaw": 3.0, "sensor_pose_of": 4.0}

f64 = np.float64
PI = f64(3.14159265358979323846)
KT_PI, KT_2PI = 3.14159265358979323846, 6.28318530717958647692


def _cr(fn, x):
    with mpmath.workdps(60):
        v = fn(mpmath.mpf(float(x)))
    with mpmath.workprec(53):  # round to nearest double
        return f64(float(+v))


def csin(x):
    return f64(math.sin(x)) if x == 0 or not math.isfinite(x) else _cr(mpmath.sin, x)


def ccos(x):
    return f64(math.cos(x)) if not math.isfinite(x) else _cr(mpmath.cos, x)


def casin(x):
    return f64(math.asin(x)) if x == 0 or abs(x) >= 1 or math.isnan(x) else _cr(mpmath.asin, x)


def catan2(y, x):
    y, x = float(y), float(x)
    if y == 0 or x == 0 or not (math.isfinite(y) and math.isfinite(x)):
        return f64(math.atan2(y, x)) if not (math.isnan(y) or math.isnan(x)) else f64("nan")
    with mpmath.workdps(60):
        v = mpmath.atan2(mpmath.mpf(y), mpmath.mpf(x))
    with mpmath.workprec(53):
        return f64(float(+v))


def set_rpy(r, p, y):
    hy, hp, hr = y * f64(0.5), p * f64(0.5), r * f64(0.5)
    cy, sy, cp, sp, cr, sr = ccos(hy), csin(hy), ccos(hp), csin(hp), ccos(hr), csin(hr)
    return [sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
            cr * cp * cy + sr * sp * sy]


def get_rpy(m):
    if abs(m[6]) >= 1:
        yaw = f64(0.0)
        delta = catan2(m[1], m[2])
        if m[6] > 0:
            return [-yaw + catan2(-m[1], -m[2]), -PI / f64(2), yaw]
        return [yaw + delta, PI / f64(2), yaw]
    pitch = -casin(m[6])
    c = ccos(pitch)
    return [catan2(m[7] / c, m[8] / c), pitch, catan2(m[3] / c, m[0] / c)]


def set_rotation(q):
    d = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    s = f64(2.0) / d
    xs, ys, zs = q[0] * s, q[1] * s, q[2] * s
    wx, wy, wz = q[3] * xs, q[3] * ys, q[3] * zs
    xx, xy, xz = q[0] * xs, q[0] * ys, q[0] * zs
    yy, yz, zz = q[1] * ys, q[1] * zs, q[2] * zs
    one = f64(1.0)
    return [one - (yy + zz), xy - wz, xz + wy, xy + wz, one - (xx + zz), yz - wx, xz - wy, yz + wx, one - (xx + yy)]


def tf2_get_yaw(q):
    x, y, z, w = q[0], q[1], q[2], q[3]
    sqx, sqy, sqz, sqw = x * x, y * y, z * z, w * w
    sarg = f64(-2) * (x * z - w * y) / (sqx + sqy + sqz + sqw)
    if sarg <= -0.99999:
        return f64(-2) * catan2(y, x)
    if sarg >= 0.99999:
        return f64(2) * catan2(y, x)
    return catan2(f64(2) * (x * y + w * z), sqw + sqx - sqy - sqz)


def normalize_angle(a):
    a = f64(a)
    while a < -KT_PI:
        a = a + f64(int(a / -KT_2PI)) * f64(KT_2PI) if a < -KT_2PI else a + f64(KT_2PI)
    while a > KT_PI:
        a = a - f64(int(a / KT_2PI)) * f64(KT_2PI) if a > KT_2PI else a - f64(KT_2PI)
    return a


def sensor_pose(robot, off):
    if robot[0] == 0 and robot[1] == 0 and robot[2] == 0:
        m = [f64(1), f64(0), f64(0), f64(0), f64(1), f64(0)]
        tx = ty = th = f64(0)
    else:
        radians = robot[2] - f64(0.0)
        c, s = ccos(radians), csin(radians)
        omc = f64(1.0) - c
        z, one = f64(0.0), f64(1.0)
        m = [z * omc + c, z * z * omc - one * s, z * one * omc + z * s,
             z * z * omc + one * s, z * omc + c, z * one * omc - z * s]
        tx, ty, th = robot[0], robot[1], robot[2] - f64(0.0)
    rx = m[0] * off[0] + m[1] * off[1] + m[2] * off[2]
    ry = m[3] * off[0] + m[4] * off[1] + m[5] * off[2]
    return [tx + rx, ty + ry, normalize_angle(off[2] + th)]


def reference(op, x):
    if op == OP_SET_RPY:
        return set_rpy(x[0], x[1], x[2])
    if op == OP_GET_RPY:
        return get_rpy(x[:9])
    if op == OP_TF_GET_YAW:
        return [get_rpy(set_rotation(x[:4]))[2]]
    if op == OP_TF2_GET_YAW:
        return [tf2_get_yaw(x[:4])]
    return sensor_pose(x[:3], x[3:6])


def units(op, k, ref, x):
    """the unit of one output's error"""
    if op == OP_SET_RPY:
        return math.ulp(max(abs(ref), 1.0))
    if op == OP_SENSOR_POSE:
        return math.ulp(max(abs(ref), abs(float(x[3])) + abs(float(x[4])))) if k < 2 else math.ulp(abs(ref))
    return math.ulp(abs(ref))


def measure(path, with_device=True):
    """-> {name: {"records", "host_max", "device_max", "host_worst", "device_worst"}}: the largest error of each side in
    the units above (inf where one side is NaN and the other not), and the record it was found on"""
    rows = np.fromfile(path, dtype=np.float64).reshape(-1, 18)
    out = {}
    with np.errstate(all="ignore"):
        for row in rows:
            op = int(row[0])
            x = [f64(v) for v in row[1:10]]
            ref = reference(op, x)
            st = out.setdefault(NAMES[op], {"records": 0, "host_max": 0.0, "device_max": 0.0, "host_worst": None,
                                            "device_worst": None, "heading_max": 0.0})
            st["records"] += 1
            for side, col in (("host", 14), ("device", 10)):
                if side == "device" and not with_device:
                    continue
                for k in range(N_OUT[op]):
                    got, r = float(row[col + k]), float(ref[k])
                    if (math.isnan(got) and math.isnan(r)) or got == r:
                        e = 0.0
                    elif math.isnan(got) or math.isnan(r) or math.isinf(got) or math.isinf(r):
                        e = math.inf
                    else:
                        e = abs(got - r) / units(op, k, r, x)
                    key = "heading_max" if op == OP_SENSOR_POSE and k == 2 else side + "_max"
                    if e > st[key]:
                        st[key] = e
                        if key != "heading_max":
                            st[side + "_worst"] = [float(v) for v in row[1:10]] + [k]
    return out
