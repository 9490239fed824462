// TEST INFRASTRUCTURE — nav_msgs/Odometry with the fields of the ROS message definition (oracle/ref_lesson5.cpp).
#pragma once

#include <memory>
#include <string>

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace nav_msgs {
struct Odometry {
  std_msgs::Header header;
  std::string child_frame_id;
  geometry_msgs::PoseWithCovariance pose;
  geometry_msgs::TwistWithCovariance twist;
  typedef std::shared_ptr<const Odometry> ConstPtr;
};
}  // namespace nav_msgs
