// TEST INFRASTRUCTURE, NOT tf — tf::Matrix3x3 (built from a quaternion, getRPY) for compiling lesson5's
// lidar_undistortion.cc and lesson6's karto_slam.cc unmodified: the tf2 stand-in under tf's name.  tf is not in the
// reference tree, so these lines stay unpinned: the de-skew tests take the roll / pitch / yaw they produce as their input.
#pragma once

#include "tf/LinearMath/Quaternion.h"

namespace tf {
typedef tf2::Matrix3x3 Matrix3x3;
}  // namespace tf
