// TEST INFRASTRUCTURE, NOT tf — tf::Quaternion for compiling lesson5's lidar_undistortion.cc and lesson6's karto_slam.cc
// unmodified.  tf's LinearMath is the same Bullet code as tf2's, so this is the tf2 stand-in under tf's name.
#pragma once

#include "tf2/LinearMath/Transform.h"

namespace tf {
typedef double tfScalar;
typedef tf2::Quaternion Quaternion;
}  // namespace tf
