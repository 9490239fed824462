/*
 * ref_lesson4_hector.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson4 Hector make-map node, reference/lesson4/src/hector_mapping/
 * hector_mapping.cc, #included where it lies (oracle/recipes.py builds it into _ref/liblesson4_ref.so).  ROS and
 * Eigen are absent; the stand-ins under oracle/shim/ (the ROS core, LaserScan, OccupancyGrid, MapMetaData, the Eigen
 * stand-in) provide the message types, the private node handle and its
 * parameters and the fixed-size Eigen types.  The node's main() is renamed so the library has none; every line of
 * ScanCallback that runs here is the reference's.
 *
 * This translation unit is compiled apart from the GMapping driver: GMapping's utils/point.h includes <math.h>, which
 * would bring std::cos(float) into the global namespace and change which `cos` the node's float-angle call resolves to.
 */
#include <chrono>
#include <cstring>
#include <iostream>
#include <memory>
#include <mutex>
#include <vector>

#include <ros/ros.h>
#include <sensor_msgs/LaserScan.h>
#include <nav_msgs/OccupancyGrid.h>

#define main lesson4_hector_mapping_main
#include "lesson4/src/hector_mapping/hector_mapping.cc"
#undef main

namespace {
hector_mapping::HectorMapping *node = nullptr;
}

extern "C" {

/* A fresh node with the parameters ref_l4_param set (shared with the GMapping driver). */
void ref_l4_hector_new(void) {
  delete node;
  std::cout.setstate(std::ios::failbit);  // the node prints its timing on every callback
  node = new hector_mapping::HectorMapping();
}

/* ScanCallback on one LaserScan.  fields[4] = angle_min, angle_increment, range_min, range_max.  info[2] = the
 * published width, height; out [width*height] = its data.  Returns 0, or -2 when nothing was published. */
int ref_l4_hector_scan(const float fields[4], int n, const float *ranges, int32_t info[2], int8_t *out, long out_cap) {
  sensor_msgs::LaserScan msg;
  msg.header.frame_id = "laser";
  msg.angle_min = fields[0];
  msg.angle_increment = fields[1];
  msg.angle_max = fields[0] + (n - 1) * fields[1];
  msg.range_min = fields[2];
  msg.range_max = fields[3];
  msg.ranges.assign(ranges, ranges + n);
  const unsigned long before = ros::shim::publish_count();
  node->ScanCallback(msg);
  if (ros::shim::publish_count() == before) return -2;
  const nav_msgs::OccupancyGrid &pub = ros::shim::last_published<nav_msgs::OccupancyGrid>();
  info[0] = (int32_t)pub.info.width;
  info[1] = (int32_t)pub.info.height;
  if ((long)pub.data.size() > out_cap) return -3;
  std::memcpy(out, pub.data.data(), pub.data.size());
  return 0;
}

}  // extern "C"
