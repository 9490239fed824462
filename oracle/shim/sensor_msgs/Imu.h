// TEST INFRASTRUCTURE — sensor_msgs/Imu with the fields of the ROS message definition (oracle/ref_lesson5.cpp).
#pragma once

#include <memory>

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace sensor_msgs {
struct Imu {
  std_msgs::Header header;
  geometry_msgs::Quaternion orientation;
  double orientation_covariance[9] = {};
  geometry_msgs::Vector3 angular_velocity;
  double angular_velocity_covariance[9] = {};
  geometry_msgs::Vector3 linear_acceleration;
  double linear_acceleration_covariance[9] = {};
  typedef std::shared_ptr<const Imu> ConstPtr;
};
}  // namespace sensor_msgs
