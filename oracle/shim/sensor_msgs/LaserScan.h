// TEST INFRASTRUCTURE — sensor_msgs/LaserScan and std_msgs/Header with the fields of the ROS message definitions, for
// compiling lesson1's feature_detection.cc unmodified (oracle/ref_lesson1.cpp).
#pragma once

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace std_msgs {
struct Header {
  uint32_t seq = 0;
  struct {
    uint32_t sec = 0, nsec = 0;
    double toSec() const { return (double)sec + 1e-9 * (double)nsec; }  // ros::Time::toSec
  } stamp;
  std::string frame_id;
};
}  // namespace std_msgs

namespace sensor_msgs {
struct LaserScan {
  std_msgs::Header header;
  float angle_min = 0, angle_max = 0, angle_increment = 0, time_increment = 0, scan_time = 0;
  float range_min = 0, range_max = 0;
  std::vector<float> ranges, intensities;
  typedef std::shared_ptr<const LaserScan> ConstPtr;
};
}  // namespace sensor_msgs
