/*
 * ref_lesson4_slam.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around lesson4's UNMODIFIED Hector SLAM node, reference/lesson4/src/hector_mapping/hector_slam.cc,
 * #included where it lies (oracle/recipes.py builds _ref/liblesson4_slam_ref.so).  ROS, tf, laser_geometry and
 * Boost are absent.  The stand-ins are, first on the include path, oracle/shim_lesson4_slam/ (laser_geometry's
 * projection, PoseStamped / PoseWithCovarianceStamped, tf's poseMsgToTF, lookupTransform and a broadcaster hook,
 * boost::lexical_cast and mutex), then oracle/shim_lesson6/ (tf's listener and types, Boost's bind / mutex / thread) and
 * oracle/shim/ (the ROS core, the messages, tf's LinearMath, the Eigen stand-in).  The node's main() is renamed; every
 * line of the node that runs here is the reference's.
 *
 * Its own translation unit: which cos / sin PoseInfoContainer's unqualified calls bind to depends on what the TU
 * includes (DESIGN.md §7).  Three things are done around the node:
 *   - its header is included with `private` / `protected` spelled `public`, after every header it pulls in, so that
 *     the driver reaches publishMap and the node's state (as ref_lesson6.cpp does);
 *   - the node's `ros::Time(0)` (a latest-time lookup) is spelled through ref_l4s_time, because the roscpp stand-in has
 *     no one-argument Time constructor;
 *   - roscpp's WallTime / WallDuration (the node's optional timing print) and ServiceServer are declared here.
 * boost::thread runs publishMapLoop once at construction; ros::ok() is false, so it returns without publishing, and the
 * driver calls publishMap itself on the library's schedule.
 */
#include <cstring>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include <ros/ros.h>
#include <boost/thread.hpp>
#include <boost/lexical_cast.hpp>
#include <tf/transform_listener.h>
#include <tf/transform_broadcaster.h>
#include <tf/transform_datatypes.h>
#include <sensor_msgs/LaserScan.h>
#include <sensor_msgs/PointCloud2.h>
#include <std_msgs/String.h>
#include <nav_msgs/GetMap.h>
#include <nav_msgs/Odometry.h>
#include <geometry_msgs/PoseStamped.h>
#include <geometry_msgs/PoseWithCovarianceStamped.h>
#include <laser_geometry/laser_geometry.h>

namespace ros {
struct WallDuration {
  double toSec() const { return 0.0; }
};
struct WallTime {
  static WallTime now() { return WallTime(); }
  WallDuration operator-(const WallTime &) const { return WallDuration(); }
};
struct ServiceServer {};
}  // namespace ros

#include "map/GridMap.h"
#include "slam_main/HectorSlamProcessor.h"
#include "scan/DataPointContainer.h"
#include "util/MapLockerInterface.h"
#include "util/HectorMapMutex.h"
#include "util/PoseInfoContainer.h"

#define private public
#define protected public
#include "lesson4/hector_mapping/hector_slam.h"
#undef private
#undef protected

inline ros::Time ref_l4s_time(int) { return ros::Time(0u, 0u); }
#define Time(x) Time(ref_l4s_time(x))
#define main lesson4_hector_slam_main
#include "lesson4/src/hector_mapping/hector_slam.cc"
#undef main
#undef Time

namespace {

HectorMappingRos *node = nullptr;

struct Captured {
  nav_msgs::Odometry odom;
  int n_odom = 0;
  std::vector<tf::StampedTransform> tfs;
  nav_msgs::OccupancyGrid map;
  int n_map = 0;
};
Captured cap;

void transform_row(const tf::Transform &t, double *out) {
  const tf::Vector3 o = t.getOrigin();
  out[0] = o.x(); out[1] = o.y(); out[2] = o.z();
  const tf::Quaternion q = t.getRotation();
  out[3] = q.x(); out[4] = q.y(); out[5] = q.z(); out[6] = q.w();
}

}  // namespace

extern "C" {

void ref_l4s_clear_params(void) { ros::shim::params().clear(); }
void ref_l4s_param(const char *name, double v) { ros::shim::params()[name] = v; }

/* A fresh node with the parameters set; mount = base_link <- laser (translation xyz + quaternion xyzw), what the
 * listener answers in the constructor. */
void ref_l4s_new(const double mount[7]) {
  delete node;
  node = nullptr;
  std::cout.setstate(std::ios::failbit);  // the node prints its timing on every callback
  tf::shim::frames().base_laser = tf::Transform(tf::Quaternion(mount[3], mount[4], mount[5], mount[6]),
                                                tf::Vector3(mount[0], mount[1], mount[2]));
  ros::shim::on_publish<nav_msgs::Odometry>() = [](const nav_msgs::Odometry &m) { cap.odom = m; cap.n_odom++; };
  ros::shim::on_publish<nav_msgs::OccupancyGrid>() = [](const nav_msgs::OccupancyGrid &m) { cap.map = m; cap.n_map++; };
  tf::shim::on_send_transform() = [](const tf::StampedTransform &t) { cap.tfs.push_back(t); };
  node = new HectorMappingRos();
}

/* scanCallback on one LaserScan.  fields[4] = angle_min, angle_increment, range_min, range_max; stamp = (sec, nsec).
 * Out: pose[3] = getLastScanMatchPose, msg[7] = odom_hector's pose (xyz + quaternion xyzw), cov[36] its covariance,
 * tfs[2][7] = the two transforms sent (map -> odom, odom -> base_link: origin + getRotation), n_points = the
 * DataContainer's size.  Returns 0, or -1 when the node did not publish one odometry message and two transforms. */
int ref_l4s_scan(const float fields[4], int n, const float *ranges, const uint32_t stamp[2], float pose[3], double msg[7],
                 double cov[36], double tfs[14], int32_t *n_points) {
  sensor_msgs::LaserScan scan;
  scan.header.frame_id = "front_laser_link";
  scan.header.stamp.sec = stamp[0];
  scan.header.stamp.nsec = stamp[1];
  scan.angle_min = fields[0];
  scan.angle_increment = fields[1];
  scan.angle_max = fields[0] + (n - 1) * fields[1];
  scan.range_min = fields[2];
  scan.range_max = fields[3];
  scan.ranges.assign(ranges, ranges + n);
  cap.n_odom = 0;
  cap.tfs.clear();
  node->scanCallback(scan);
  if (cap.n_odom != 1 || cap.tfs.size() != 2) return -1;
  const Eigen::Vector3f p = node->slamProcessor->getLastScanMatchPose();
  pose[0] = p.x(); pose[1] = p.y(); pose[2] = p.z();
  const geometry_msgs::Pose &m = cap.odom.pose.pose;
  msg[0] = m.position.x; msg[1] = m.position.y; msg[2] = m.position.z;
  msg[3] = m.orientation.x; msg[4] = m.orientation.y; msg[5] = m.orientation.z; msg[6] = m.orientation.w;
  for (int i = 0; i < 36; i++) cov[i] = cap.odom.pose.covariance[i];
  transform_row(cap.tfs[0], tfs);
  transform_row(cap.tfs[1], tfs + 7);
  *n_points = (int32_t)node->laserScanContainer.getSize();
  return 0;
}

/* publishMap of level 0 stamped (sec, nsec), as publishMapLoop calls it.  info[5] = origin x, origin y, resolution,
 * width, height; out = the payload (capacity out_cap); *rebuilt = 1 when the update-index gate rebuilt it.  Returns 0,
 * -1 when nothing was published, -2 when out is too small. */
int ref_l4s_publish(const uint32_t stamp[2], double info[5], int8_t *out, long out_cap, int32_t *rebuilt) {
  const int before = node->lastGetMapUpdateIndex;
  const int index = node->slamProcessor->getGridMap(0).getUpdateIndex();
  cap.n_map = 0;
  node->publishMap(node->mapPubContainer[0], node->slamProcessor->getGridMap(0), ros::Time(stamp[0], stamp[1]),
                   node->slamProcessor->getMapMutex(0));
  if (cap.n_map != 1) return -1;
  const nav_msgs::OccupancyGrid &g = cap.map;
  if (g.header.stamp.sec != stamp[0] || g.header.stamp.nsec != stamp[1]) return -3;
  info[0] = g.info.origin.position.x;
  info[1] = g.info.origin.position.y;
  info[2] = g.info.resolution;
  info[3] = g.info.width;
  info[4] = g.info.height;
  if ((long)g.data.size() > out_cap) return -2;
  std::memcpy(out, g.data.data(), g.data.size());
  *rebuilt = before != index ? 1 : 0;
  return 0;
}

}  // extern "C"
