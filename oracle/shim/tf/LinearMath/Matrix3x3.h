// TEST INFRASTRUCTURE, NOT tf — tf::Matrix3x3 built from a quaternion, and getRPY, restated from tf's published
// LinearMath algorithms (Matrix3x3::setRotation and getEulerYPR, solution 1) for compiling lesson5's
// lidar_undistortion.cc unmodified (oracle/ref_lesson5.cpp).  tf is not in the reference tree, so these lines stay
// unpinned: the de-skew tests take the roll / pitch / yaw this stand-in produces as their input.
#pragma once

#include <cmath>

#include "tf/LinearMath/Quaternion.h"

namespace tf {
class Matrix3x3 {
 public:
  explicit Matrix3x3(const Quaternion &q) {
    const tfScalar d = q.length2(), s = tfScalar(2.0) / d;
    const tfScalar xs = q.x() * s, ys = q.y() * s, zs = q.z() * s;
    const tfScalar wx = q.w() * xs, wy = q.w() * ys, wz = q.w() * zs;
    const tfScalar xx = q.x() * xs, xy = q.x() * ys, xz = q.x() * zs;
    const tfScalar yy = q.y() * ys, yz = q.y() * zs, zz = q.z() * zs;
    set(0, tfScalar(1.0) - (yy + zz), xy - wz, xz + wy);
    set(1, xy + wz, tfScalar(1.0) - (xx + zz), yz - wx);
    set(2, xz - wy, yz + wx, tfScalar(1.0) - (xx + yy));
  }
  // R = Rz(yaw) Ry(pitch) Rx(roll); at the pitch singularity yaw is 0 and roll takes the whole turn
  void getRPY(tfScalar &roll, tfScalar &pitch, tfScalar &yaw) const {
    if (std::fabs(m_[2][0]) >= 1) {
      yaw = 0;
      const tfScalar delta = std::atan2(m_[0][1], m_[0][2]);
      if (m_[2][0] > 0) {
        pitch = -M_PI / 2;
        roll = -yaw + std::atan2(-m_[0][1], -m_[0][2]);
      } else {
        pitch = M_PI / 2;
        roll = yaw + delta;
      }
      return;
    }
    pitch = -std::asin(m_[2][0]);
    const tfScalar c = std::cos(pitch);
    roll = std::atan2(m_[2][1] / c, m_[2][2] / c);
    yaw = std::atan2(m_[1][0] / c, m_[0][0] / c);
  }

 private:
  void set(int r, tfScalar a, tfScalar b, tfScalar c) { m_[r][0] = a; m_[r][1] = b; m_[r][2] = c; }
  tfScalar m_[3][3];
};
}  // namespace tf
