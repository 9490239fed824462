// TEST INFRASTRUCTURE — geometry_msgs/PoseStamped with the fields of the ROS message definition (oracle/ref_lesson4_slam.cpp).
#pragma once

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace geometry_msgs {
struct PoseStamped {
  std_msgs::Header header;
  Pose pose;
};
}  // namespace geometry_msgs
