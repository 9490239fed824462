// TEST INFRASTRUCTURE — tf2_ros Buffer / TransformListener for lesson3's plicp_odometry.cc (oracle/ref_lesson3.cpp):
// lookupTransform answers with the laser mount the driver sets (tf2_ros::shim::mount()), for any frames.
#pragma once

#include <stdexcept>
#include <string>

#include "geometry_msgs/TransformStamped.h"
#include "ros/ros.h"

namespace tf2 {
struct TransformException : std::runtime_error {
  using std::runtime_error::runtime_error;
};
}  // namespace tf2

namespace tf2_ros {
namespace shim {
inline geometry_msgs::Transform &mount() {
  static geometry_msgs::Transform t;
  return t;
}
}  // namespace shim

struct Buffer {
  geometry_msgs::TransformStamped lookupTransform(const std::string &, const std::string &, const ros::Time &,
                                                  const ros::Duration &) const {
    geometry_msgs::TransformStamped m;
    m.transform = shim::mount();
    return m;
  }
};
struct TransformListener {
  explicit TransformListener(Buffer &) {}
};
}  // namespace tf2_ros
