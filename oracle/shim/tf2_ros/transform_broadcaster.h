// TEST INFRASTRUCTURE — tf2_ros TransformBroadcaster for lesson3's plicp_odometry.cc: the transform is dropped (the
// odometry message carries the same pose).
#pragma once

#include "geometry_msgs/TransformStamped.h"

namespace tf2_ros {
struct TransformBroadcaster {
  void sendTransform(const geometry_msgs::TransformStamped &) {}
};
}  // namespace tf2_ros
