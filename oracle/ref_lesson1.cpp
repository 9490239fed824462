/*
 * ref_lesson1.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson1 node, reference/lesson1/src/feature_detection.cc, #included where it
 * lies (oracle/recipes.py builds _ref/liblesson1_ref.so).  ROS is absent; oracle/shim/ros/ros.h and
 * oracle/shim/sensor_msgs/LaserScan.h stand in for the message types and the node handle.  The node's main() is
 * renamed so the library has none; every line of LaserScan::ScanCallback (:77-179) that runs here is the reference's.
 */
#include <cstring>

#define main lesson1_feature_detection_main
#include "lesson1/src/feature_detection.cc"
#undef main

extern "C" {

/* ScanCallback on one scan of n ranges (n <= max_scan_count); out[1500] = the published corner_scan.ranges.
 * Returns 0, or -1 where the node would overflow new_scan (n > 1500). */
int ref_feature_detect(int n, const float *ranges, float *out) {
  if (n < 0 || n > max_scan_count) return -1;
  static LaserScan *node = new LaserScan();  // edge_threshold_ = 1.0 (:69); the node keeps no state between scans
  auto msg = std::make_shared<sensor_msgs::LaserScan>();
  msg->ranges.assign(ranges, ranges + n);
  sensor_msgs::LaserScan::ConstPtr cmsg = msg;
  node->ScanCallback(cmsg);
  const sensor_msgs::LaserScan &pub = ros::shim::last_published<sensor_msgs::LaserScan>();
  if ((int)pub.ranges.size() != max_scan_count) return -2;
  std::memcpy(out, pub.ranges.data(), sizeof(float) * max_scan_count);
  return 0;
}

int ref_feature_max_beams(void) { return max_scan_count; }

}  // extern "C"
