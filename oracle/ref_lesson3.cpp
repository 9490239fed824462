/*
 * ref_lesson3.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson3 odometry node, reference/lesson3/src/plicp_odometry.cc, #included
 * where it lies (oracle/recipes.py builds _ref/liblesson3_ref.so).  ROS, tf2 and CSM are absent; the stand-ins under
 * oracle/shim/ provide the message types, the node handle and its parameters, ros::Time, tf2's LinearMath, the tf2_ros
 * buffer (answering with the mount the driver sets) and CSM's types with sm_icp answered by orc_plicp_match
 * (oracle/plicp_oracle.c, linked in).  The node's main() is renamed so the library has none; every line of the node's
 * callback that runs here is the reference's.  LaserScans go in through the public ScanCallback; the published odometry
 * and the state it came from (input_.first_guess, output_, whether prev_ldp_scan_ was replaced) come back out.
 *
 * The node's header is included with `private` spelled `public`, after every other header it pulls in, so that only
 * the node's class is affected.
 */
#include <cstring>
#include <memory>
#include <vector>

#include <ros/ros.h>
#include <sensor_msgs/LaserScan.h>
#include <geometry_msgs/TwistStamped.h>
#include <geometry_msgs/TransformStamped.h>
#include <nav_msgs/Odometry.h>
#include <tf2/utils.h>
#include <tf2/LinearMath/Transform.h>
#include <tf2_ros/transform_listener.h>
#include <tf2_ros/transform_broadcaster.h>
#include <tf2_geometry_msgs/tf2_geometry_msgs.h>
#include <csm/csm_all.h>

#define private public
#include <lesson3/plicp_odometry.h>
#undef private

#define main lesson3_plicp_odometry_main
#include "lesson3/src/plicp_odometry.cc"
#undef main

namespace {
ScanMatchPLICP *node = nullptr;
}

extern "C" {

/* clear the parameter server; ref_plicp_param sets one value; ref_plicp_new makes a fresh node with them and the laser
 * mount translation xyz + quaternion xyzw */
void ref_plicp_clear_params() { ros::shim::params().clear(); }
void ref_plicp_param(const char *name, double value) { ros::shim::params()[name] = value; }

void ref_plicp_new(const double mount[7]) {
  delete node;
  auto &m = tf2_ros::shim::mount();
  m.translation.x = mount[0]; m.translation.y = mount[1]; m.translation.z = mount[2];
  m.rotation.x = mount[3]; m.rotation.y = mount[4]; m.rotation.z = mount[5]; m.rotation.w = mount[6];
  node = new ScanMatchPLICP();
}

/* ScanCallback on one LaserScan; fields[4] = angle_min, angle_increment, range_min, range_max.  out = one
 * b2s_plicp_odom_step (reference_scan is left 0: the caller tracks it).  Returns 0, or -1 when the callback threw. */
int ref_plicp_scan(uint32_t sec, uint32_t nsec, const float fields[4], int n, const float *ranges,
                   b2s_plicp_odom_step *out) {
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
  const unsigned long before = ros::shim::publish_count();
  const LDP kf_before = node->initialized_ ? node->prev_ldp_scan_ : nullptr;
  try {
    node->ScanCallback(c);
  } catch (const std::exception &) {
    return -1;
  }
  std::memset(out, 0, sizeof *out);
  out->published = ros::shim::publish_count() != before;
  out->keyframe = node->prev_ldp_scan_ != kf_before;
  if (!out->published) {
    out->orientation[3] = 1.0;
    out->reference_scan = -1;
    return 0;
  }
  const nav_msgs::Odometry &o = ros::shim::last_published<nav_msgs::Odometry>();
  out->position[0] = o.pose.pose.position.x;
  out->position[1] = o.pose.pose.position.y;
  out->position[2] = o.pose.pose.position.z;
  out->orientation[0] = o.pose.pose.orientation.x;
  out->orientation[1] = o.pose.pose.orientation.y;
  out->orientation[2] = o.pose.pose.orientation.z;
  out->orientation[3] = o.pose.pose.orientation.w;
  out->linear[0] = o.twist.twist.linear.x;
  out->linear[1] = o.twist.twist.linear.y;
  out->linear[2] = o.twist.twist.linear.z;
  out->angular[0] = o.twist.twist.angular.x;
  out->angular[1] = o.twist.twist.angular.y;
  out->angular[2] = o.twist.twist.angular.z;
  for (int k = 0; k < 3; k++) out->first_guess[k] = node->input_.first_guess[k];
  for (int k = 0; k < 3; k++) out->icp.x[k] = node->output_.x[k];
  out->icp.valid = node->output_.valid;
  out->icp.iterations = node->output_.iterations;
  out->icp.nvalid = node->output_.nvalid;
  out->icp.error = node->output_.error;
  return 0;
}

}  // extern "C"
