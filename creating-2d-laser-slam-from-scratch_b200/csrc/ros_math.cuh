// The ROS plumbing the ported nodes compute with: tf / tf2 LinearMath (Bullet's Matrix3x3, Quaternion, Transform) and
// roscpp's Time / Duration, restated from their published code operation by operation in double / integer arithmetic.
// tf and roscpp are not in the reference tree, so this arithmetic is unpinned (DESIGN.md §7): the test infrastructure
// states it twice more, in the stand-ins the unmodified nodes build against and in the C restatements, and
// tests/ros_math_check.cpp holds the three equal bit for bit.  Quaternions are double[4] (x, y, z, w).
// Keep every expression in its order: device code builds with -fmad=false, and the x86-64 host has no FMA to contract
// to.  Host + device code, like glibc_math.cuh: no CUDA runtime include, so g++ compiles it for the CPU test.
#pragma once

#include <math.h>
#include <stdint.h>

#ifndef B2S_HD
#if defined(__CUDACC__)
#define B2S_HD __host__ __device__ __forceinline__
#else
#define B2S_HD static inline
#endif
#endif

namespace b2s {

// tf2::Transform: basis rows and origin
struct TfTransform {
  double m[3][3];
  double o[3];
};

B2S_HD void tf_identity(TfTransform &t) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) t.m[i][j] = i == j ? 1.0 : 0.0;
    t.o[i] = 0.0;
  }
}

// Transform::operator()(v): v.dot3(basis rows) + origin
B2S_HD void tf_apply(const TfTransform &t, const double v[3], double out[3]) {
  for (int i = 0; i < 3; i++) out[i] = (v[0] * t.m[i][0] + v[1] * t.m[i][1] + v[2] * t.m[i][2]) + t.o[i];
}

// Transform::operator* : (basis1 * basis2, transform1(origin2)); the Matrix3x3 product through tdotx / tdoty / tdotz
B2S_HD TfTransform tf_mul(const TfTransform &a, const TfTransform &b) {
  TfTransform c;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) c.m[i][j] = b.m[0][j] * a.m[i][0] + b.m[1][j] * a.m[i][1] + b.m[2][j] * a.m[i][2];
    c.o[i] = (b.o[0] * a.m[i][0] + b.o[1] * a.m[i][1] + b.o[2] * a.m[i][2]) + a.o[i];
  }
  return c;
}

// Transform::inverse : (basis^T, basis^T * -origin)
B2S_HD TfTransform tf_inverse(const TfTransform &a) {
  TfTransform c;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) c.m[i][j] = a.m[j][i];
  const double no[3] = {-a.o[0], -a.o[1], -a.o[2]};
  for (int i = 0; i < 3; i++) c.o[i] = c.m[i][0] * no[0] + c.m[i][1] * no[1] + c.m[i][2] * no[2];
  return c;
}

// Matrix3x3::setRotation(q)
B2S_HD void tf_set_rotation(TfTransform &t, const double q[4]) {
  const double d = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  const double s = 2.0 / d;
  const double xs = q[0] * s, ys = q[1] * s, zs = q[2] * s;
  const double wx = q[3] * xs, wy = q[3] * ys, wz = q[3] * zs;
  const double xx = q[0] * xs, xy = q[0] * ys, xz = q[0] * zs;
  const double yy = q[1] * ys, yz = q[1] * zs, zz = q[2] * zs;
  t.m[0][0] = 1.0 - (yy + zz); t.m[0][1] = xy - wz; t.m[0][2] = xz + wy;
  t.m[1][0] = xy + wz; t.m[1][1] = 1.0 - (xx + zz); t.m[1][2] = yz - wx;
  t.m[2][0] = xz - wy; t.m[2][1] = yz + wx; t.m[2][2] = 1.0 - (xx + yy);
}

// Matrix3x3::getRotation(q)
B2S_HD void tf_get_rotation(const TfTransform &t, double q[4]) {
  const double trace = t.m[0][0] + t.m[1][1] + t.m[2][2];
  if (trace > 0.0) {
    double s = sqrt(trace + 1.0);
    q[3] = s * 0.5;
    s = 0.5 / s;
    q[0] = (t.m[2][1] - t.m[1][2]) * s;
    q[1] = (t.m[0][2] - t.m[2][0]) * s;
    q[2] = (t.m[1][0] - t.m[0][1]) * s;
  } else {
    const int i = t.m[0][0] < t.m[1][1] ? (t.m[1][1] < t.m[2][2] ? 2 : 1) : (t.m[0][0] < t.m[2][2] ? 2 : 0);
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = sqrt(t.m[i][i] - t.m[j][j] - t.m[k][k] + 1.0);
    q[i] = s * 0.5;
    s = 0.5 / s;
    q[3] = (t.m[k][j] - t.m[j][k]) * s;
    q[j] = (t.m[j][i] + t.m[i][j]) * s;
    q[k] = (t.m[k][i] + t.m[i][k]) * s;
  }
}

// Quaternion::setRPY (tf::createQuaternionFromRPY)
B2S_HD void quat_set_rpy(double roll, double pitch, double yaw, double q[4]) {
  const double hy = yaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
  const double cy = cos(hy), sy = sin(hy), cp = cos(hp), sp = sin(hp), cr = cos(hr), sr = sin(hr);
  q[0] = sr * cp * cy - cr * sp * sy;
  q[1] = cr * sp * cy + sr * cp * sy;
  q[2] = cr * cp * sy - sr * sp * cy;
  q[3] = cr * cp * cy + sr * sp * sy;
}

// tf's Matrix3x3::getRPY: getEulerYPR, solution 1.  At the pitch singularity yaw is 0 and roll takes the whole turn.
B2S_HD void tf_get_rpy(const TfTransform &t, double &roll, double &pitch, double &yaw) {
  const double pi = 3.14159265358979323846;
  if (fabs(t.m[2][0]) >= 1) {
    yaw = 0;
    const double delta = atan2(t.m[0][1], t.m[0][2]);
    if (t.m[2][0] > 0) {
      pitch = -pi / 2;
      roll = -yaw + atan2(-t.m[0][1], -t.m[0][2]);
    } else {
      pitch = pi / 2;
      roll = yaw + delta;
    }
    return;
  }
  pitch = -asin(t.m[2][0]);
  const double c = cos(pitch);
  roll = atan2(t.m[2][1] / c, t.m[2][2] / c);
  yaw = atan2(t.m[1][0] / c, t.m[0][0] / c);
}

// tf::getYaw(q): the yaw of Matrix3x3(q).getRPY
B2S_HD double tf_get_yaw(const double q[4]) {
  TfTransform t;
  tf_set_rotation(t, q);
  double roll, pitch, yaw;
  tf_get_rpy(t, roll, pitch, yaw);
  return yaw;
}

// tf2::getYaw(q): the yaw of tf2::getEulerYPR (tf2/utils.h), a different formula from tf's
B2S_HD double tf2_get_yaw(const double q[4]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double sqx = x * x, sqy = y * y, sqz = z * z, sqw = w * w;
  const double sarg = -2 * (x * z - w * y) / (sqx + sqy + sqz + sqw);
  if (sarg <= -0.99999) return -2 * atan2(y, x);
  if (sarg >= 0.99999) return 2 * atan2(y, x);
  return atan2(2 * (x * y + w * z), sqw + sqx - sqy - sqz);
}

// ros::Duration: 0 <= nsec < 1e9 once normalised
struct RosDuration {
  int32_t sec, nsec;
};

// Time - Time: the (sec, nsec) differences, normalised (normalizeSecNSecSigned)
B2S_HD RosDuration ros_time_diff(uint32_t sec1, uint32_t nsec1, uint32_t sec0, uint32_t nsec0) {
  const int64_t dsec = (int64_t)(int32_t)sec1 - (int32_t)sec0, dnsec = (int64_t)(int32_t)nsec1 - (int32_t)nsec0;
  int64_t nsec_part = dnsec % 1000000000LL, sec_part = dsec + dnsec / 1000000000LL;
  if (nsec_part < 0) {
    nsec_part += 1000000000LL;
    --sec_part;
  }
  return RosDuration{(int32_t)sec_part, (int32_t)nsec_part};
}

// Duration::fromSec: floor(d) seconds and round((d - sec) * 1e9) nanoseconds, a whole second rolled over
B2S_HD RosDuration ros_duration_from_sec(double d) {
  RosDuration r;
  r.sec = (int32_t)(int64_t)floor(d);
  r.nsec = (int32_t)round((d - r.sec) * 1e9);
  r.sec += r.nsec / 1000000000;
  r.nsec %= 1000000000;
  return r;
}

// Duration's operator>: by (sec, nsec)
B2S_HD bool ros_duration_gt(const RosDuration &a, const RosDuration &b) {
  return a.sec > b.sec || (a.sec == b.sec && a.nsec > b.nsec);
}

// Duration::toSec and Time::toSec
B2S_HD double ros_duration_to_sec(const RosDuration &d) { return (double)d.sec + 1e-9 * (double)d.nsec; }
B2S_HD double ros_time_to_sec(uint32_t sec, uint32_t nsec) { return (double)sec + 1e-9 * (double)nsec; }

}  // namespace b2s
