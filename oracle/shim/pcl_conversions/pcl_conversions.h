// TEST INFRASTRUCTURE, NOT pcl_conversions — toPCL for a message header (oracle/ref_lesson5.cpp).
#pragma once

#include "pcl/point_cloud.h"
#include "sensor_msgs/LaserScan.h"

namespace pcl_conversions {
inline void toPCL(const std_msgs::Header &h, pcl::PCLHeader &out) {
  out.stamp = (uint64_t)h.stamp.sec * 1000000ull + h.stamp.nsec / 1000ull;
  out.seq = h.seq;
  out.frame_id = h.frame_id;
}
}  // namespace pcl_conversions
