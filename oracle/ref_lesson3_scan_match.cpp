/*
 * ref_lesson3_scan_match.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson3 scan-to-scan node, reference/lesson3/src/scan_match_plicp.cc,
 * #included where it lies (oracle/recipes.py builds _ref/liblesson3_scan_match_ref.so; the node's class
 * has the odometry node's name, so it gets a library of its own).  ROS and CSM are absent; the stand-ins under
 * oracle/shim/ provide the message types, the node handle and its parameters, ros::Time and CSM's types with sm_icp
 * answered by orc_plicp_match (oracle/plicp_oracle.c, linked in).  The node's main() is renamed so the library has
 * none; every line of the node's callback that runs here is the reference's.  LaserScans go in through the public
 * ScanCallback; output_ comes back out after each one.
 *
 * The node's header is included with `private` spelled `public`, after every other header it pulls in, so that only
 * the node's class is affected.
 */
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>
#include <chrono>
#include <iostream>

#include <ros/ros.h>
#include <sensor_msgs/LaserScan.h>
#include <geometry_msgs/TwistStamped.h>
#include <tf2/utils.h>
#include <tf2/LinearMath/Transform.h>
#include <tf2_ros/transform_listener.h>
#include <tf2_ros/transform_broadcaster.h>
#include <csm/csm_all.h>

#define private public
#include <lesson3/scan_match_plicp.h>
#undef private

#define main lesson3_scan_match_plicp_main
#include "lesson3/src/scan_match_plicp.cc"
#undef main

namespace {
ScanMatchPLICP *node = nullptr;
}

extern "C" {

/* clear the parameter server; ref_sm_param sets one value; ref_sm_new makes a fresh node with them */
void ref_sm_clear_params() { ros::shim::params().clear(); }
void ref_sm_param(const char *name, double value) { ros::shim::params()[name] = value; }

/* The node writes its timings and every match to std::cout (:185, :194, :288-293).  The stream is put in a failed
 * state first, so those lines format nothing: the answers are read from output_, and a library linked with its own
 * static libstdc++ crashes formatting a double through the stream's locale when it is loaded into a process that
 * already holds another libstdc++ (Python with numpy). */
void ref_sm_new() {
  std::cout.setstate(std::ios::badbit);
  delete node;
  node = new ScanMatchPLICP();
}

/* ScanCallback on one LaserScan; fields[4] = angle_min, angle_increment, range_min, range_max.  out = one
 * b2s_plicp_scan_match_step: output_ and what the node prints from it, or all zero for the scan that initialises the
 * node.  Returns 0, or -1 when the callback threw. */
int ref_sm_scan(uint32_t sec, uint32_t nsec, const float fields[4], int n, const float *ranges,
                b2s_plicp_scan_match_step *out) {
  auto m = std::make_shared<sensor_msgs::LaserScan>();
  m->header.stamp.sec = sec;
  m->header.stamp.nsec = nsec;
  m->header.frame_id = "laser";
  m->angle_min = fields[0];
  m->angle_increment = fields[1];
  m->angle_max = fields[0] + (n - 1) * fields[1];
  m->range_min = fields[2];
  m->range_max = fields[3];
  m->ranges.assign(ranges, ranges + n);
  sensor_msgs::LaserScan::ConstPtr c = m;
  const bool matches = node->initialized_;
  try {
    node->ScanCallback(c);
  } catch (const std::exception &) {
    return -1;
  }
  std::memset(out, 0, sizeof *out);
  if (!matches) return 0;
  for (int k = 0; k < 3; k++) out->icp.x[k] = node->output_.x[k];
  out->icp.valid = node->output_.valid;
  out->icp.iterations = node->output_.iterations;
  out->icp.nvalid = node->output_.nvalid;
  out->icp.error = node->output_.error;
  out->theta_deg = node->output_.x[2] * 180 / M_PI;  // the expression the node prints (:289)
  out->matched = 1;
  return 0;
}

}  // extern "C"
