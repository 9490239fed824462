// TEST INFRASTRUCTURE — tf2/utils.h getYaw: the yaw of getEulerYPR (geometry2), restated for compiling lesson3's
// plicp_odometry.cc unmodified (oracle/ref_lesson3.cpp).
#pragma once

#include <cmath>

#include "tf2/LinearMath/Transform.h"

namespace tf2 {
template <class A>
void getEulerYPR(const A &a, double &yaw, double &pitch, double &roll) {
  double sqx = a.x() * a.x(), sqy = a.y() * a.y(), sqz = a.z() * a.z(), sqw = a.w() * a.w();
  double sarg = -2 * (a.x() * a.z() - a.w() * a.y()) / (sqx + sqy + sqz + sqw);
  if (sarg <= -0.99999) {
    pitch = -0.5 * M_PI;
    roll = 0;
    yaw = -2 * atan2(a.y(), a.x());
  } else if (sarg >= 0.99999) {
    pitch = 0.5 * M_PI;
    roll = 0;
    yaw = 2 * atan2(a.y(), a.x());
  } else {
    pitch = asin(sarg);
    roll = atan2(2 * (a.y() * a.z() + a.w() * a.x()), sqw - sqx - sqy + sqz);
    yaw = atan2(2 * (a.x() * a.y() + a.w() * a.z()), sqw + sqx - sqy - sqz);
  }
}
template <class A>
double getYaw(const A &a) {
  double yaw, pitch, roll;
  getEulerYPR(a, yaw, pitch, roll);
  return yaw;
}
}  // namespace tf2
