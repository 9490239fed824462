// TEST INFRASTRUCTURE — geometry_msgs/PoseWithCovarianceStamped for lesson4's hector_slam.cc (oracle/ref_lesson4_slam.cpp).
// The node binds a boost::array<double, 36> & to its pose's covariance (PoseInfoContainer.h:72), as roscpp's generated
// messages declare it, so this message's PoseWithCovariance holds a boost::array (std::array here).  It converts to the
// double[36] form of oracle/shim/geometry_msgs/messages.h, which nav_msgs::Odometry and lesson5's build keep.
#pragma once

#include <array>
#include <cstddef>

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace boost {
template <class T, std::size_t N>
using array = std::array<T, N>;
}  // namespace boost

namespace geometry_msgs {
struct PoseWithCovarianceArray {
  Pose pose;
  boost::array<double, 36> covariance{};
  operator PoseWithCovariance() const {
    PoseWithCovariance p;
    p.pose = pose;
    for (int i = 0; i < 36; i++) p.covariance[i] = covariance[i];
    return p;
  }
};
struct PoseWithCovarianceStamped {
  std_msgs::Header header;
  PoseWithCovarianceArray pose;
};
}  // namespace geometry_msgs
