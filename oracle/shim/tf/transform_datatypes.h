// TEST INFRASTRUCTURE, NOT tf — quaternionMsgToTF for compiling lesson5's lidar_undistortion.cc unmodified
// (oracle/ref_lesson5.cpp).
#pragma once

#include "geometry_msgs/messages.h"
#include "tf/LinearMath/Matrix3x3.h"
#include "tf/LinearMath/Quaternion.h"

namespace tf {
inline void quaternionMsgToTF(const geometry_msgs::Quaternion &msg, Quaternion &q) { q = Quaternion(msg.x, msg.y, msg.z, msg.w); }
}  // namespace tf
