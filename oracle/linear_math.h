/*
 * linear_math.h — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * tf / tf2 LinearMath (Bullet's Matrix3x3, Quaternion, Transform) and roscpp's Time / Duration as the C restatements use
 * them (plicp_odometry_oracle.c, deskew_node_oracle.c), restated from the published code operation by operation in
 * double / integer arithmetic; build without FMA contraction.  Quaternions are double[4] (x, y, z, w).  The library's
 * csrc/ros_math.cuh states the same arithmetic for the device, and tests/ros_math_check.cpp holds the two equal bit for
 * bit.  The node stand-ins under oracle/shim/ do not include this header: it brings <math.h>, which decides what a
 * node's unqualified cos / sin bind to (DESIGN.md §7 (1)).
 */
#pragma once

#include <math.h>
#include <stdint.h>

/* tf2::Transform: basis rows and origin */
typedef struct { double m[3][3], o[3]; } orc_tf;

static inline void tf_identity(orc_tf *t) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) t->m[i][j] = i == j ? 1.0 : 0.0;
    t->o[i] = 0.0;
  }
}
/* Transform::operator* : (basis1 * basis2, transform1(origin2)) */
static inline orc_tf tf_mul(const orc_tf *a, const orc_tf *b) {
  orc_tf c;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) c.m[i][j] = b->m[0][j] * a->m[i][0] + b->m[1][j] * a->m[i][1] + b->m[2][j] * a->m[i][2];
    c.o[i] = (b->o[0] * a->m[i][0] + b->o[1] * a->m[i][1] + b->o[2] * a->m[i][2]) + a->o[i];
  }
  return c;
}
/* Transform::inverse : (basis^T, basis^T * -origin) */
static inline orc_tf tf_inverse(const orc_tf *a) {
  orc_tf c;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) c.m[i][j] = a->m[j][i];
  const double no[3] = {-a->o[0], -a->o[1], -a->o[2]};
  for (int i = 0; i < 3; i++) c.o[i] = c.m[i][0] * no[0] + c.m[i][1] * no[1] + c.m[i][2] * no[2];
  return c;
}
/* Matrix3x3::setRotation(q) */
static inline void tf_set_rotation(orc_tf *t, const double q[4]) {
  const double d = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3], s = 2.0 / d;
  const double xs = q[0] * s, ys = q[1] * s, zs = q[2] * s;
  const double wx = q[3] * xs, wy = q[3] * ys, wz = q[3] * zs;
  const double xx = q[0] * xs, xy = q[0] * ys, xz = q[0] * zs;
  const double yy = q[1] * ys, yz = q[1] * zs, zz = q[2] * zs;
  t->m[0][0] = 1.0 - (yy + zz); t->m[0][1] = xy - wz; t->m[0][2] = xz + wy;
  t->m[1][0] = xy + wz; t->m[1][1] = 1.0 - (xx + zz); t->m[1][2] = yz - wx;
  t->m[2][0] = xz - wy; t->m[2][1] = yz + wx; t->m[2][2] = 1.0 - (xx + yy);
}
/* Matrix3x3::getRotation(q) */
static inline void tf_get_rotation(const orc_tf *t, double q[4]) {
  const double trace = t->m[0][0] + t->m[1][1] + t->m[2][2];
  if (trace > 0.0) {
    double s = sqrt(trace + 1.0);
    q[3] = s * 0.5;
    s = 0.5 / s;
    q[0] = (t->m[2][1] - t->m[1][2]) * s;
    q[1] = (t->m[0][2] - t->m[2][0]) * s;
    q[2] = (t->m[1][0] - t->m[0][1]) * s;
  } else {
    const int i = t->m[0][0] < t->m[1][1] ? (t->m[1][1] < t->m[2][2] ? 2 : 1) : (t->m[0][0] < t->m[2][2] ? 2 : 0);
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = sqrt(t->m[i][i] - t->m[j][j] - t->m[k][k] + 1.0);
    q[i] = s * 0.5;
    s = 0.5 / s;
    q[3] = (t->m[k][j] - t->m[j][k]) * s;
    q[j] = (t->m[j][i] + t->m[i][j]) * s;
    q[k] = (t->m[k][i] + t->m[i][k]) * s;
  }
}
/* Quaternion::setRPY */
static inline void quat_set_rpy(double roll, double pitch, double yaw, double q[4]) {
  const double hy = yaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
  const double cy = cos(hy), sy = sin(hy), cp = cos(hp), sp = sin(hp), cr = cos(hr), sr = sin(hr);
  q[0] = sr * cp * cy - cr * sp * sy;
  q[1] = cr * sp * cy + sr * cp * sy;
  q[2] = cr * cp * sy - sr * sp * cy;
  q[3] = cr * cp * cy + sr * sp * sy;
}
/* tf's Matrix3x3::getRPY: getEulerYPR, solution 1; at the pitch singularity yaw is 0 and roll takes the whole turn */
static inline void tf_get_rpy(const orc_tf *t, double *roll, double *pitch, double *yaw) {
  const double pi = 3.14159265358979323846;
  if (fabs(t->m[2][0]) >= 1) {
    *yaw = 0;
    const double delta = atan2(t->m[0][1], t->m[0][2]);
    if (t->m[2][0] > 0) {
      *pitch = -pi / 2;
      *roll = -*yaw + atan2(-t->m[0][1], -t->m[0][2]);
    } else {
      *pitch = pi / 2;
      *roll = *yaw + delta;
    }
    return;
  }
  *pitch = -asin(t->m[2][0]);
  const double c = cos(*pitch);
  *roll = atan2(t->m[2][1] / c, t->m[2][2] / c);
  *yaw = atan2(t->m[1][0] / c, t->m[0][0] / c);
}
/* tf2::getYaw(q): the yaw of tf2::getEulerYPR (tf2/utils.h), a different formula from tf's */
static inline double tf2_get_yaw(const double q[4]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double sqx = x * x, sqy = y * y, sqz = z * z, sqw = w * w;
  const double sarg = -2 * (x * z - w * y) / (sqx + sqy + sqz + sqw);
  if (sarg <= -0.99999) return -2 * atan2(y, x);
  if (sarg >= 0.99999) return 2 * atan2(y, x);
  return atan2(2 * (x * y + w * z), sqw + sqx - sqy - sqz);
}

/* ros::Duration, 0 <= nsec < 1e9 once normalised */
typedef struct { int32_t sec, nsec; } orc_duration;

/* Time - Time: the (sec, nsec) differences, normalised (normalizeSecNSecSigned) */
static inline orc_duration ros_time_diff(uint32_t sec1, uint32_t nsec1, uint32_t sec0, uint32_t nsec0) {
  const long long dsec = (long long)(int32_t)sec1 - (int32_t)sec0, dnsec = (long long)(int32_t)nsec1 - (int32_t)nsec0;
  long long nsec_part = dnsec % 1000000000LL, sec_part = dsec + dnsec / 1000000000LL;
  if (nsec_part < 0) { nsec_part += 1000000000LL; --sec_part; }
  const orc_duration d = {(int32_t)sec_part, (int32_t)nsec_part};
  return d;
}
/* Duration::toSec and Time::toSec */
static inline double ros_duration_to_sec(orc_duration d) { return (double)d.sec + 1e-9 * (double)d.nsec; }
static inline double ros_time_to_sec(uint32_t sec, uint32_t nsec) { return (double)sec + 1e-9 * (double)nsec; }
