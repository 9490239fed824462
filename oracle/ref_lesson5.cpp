/*
 * ref_lesson5.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson5 node, reference/lesson5/src/lidar_undistortion.cc, #included where it
 * lies (oracle/recipes.py builds _ref/liblesson5_ref.so).  ROS, tf, PCL and Eigen are absent; the stand-ins under
 * oracle/shim/ provide the message types, the node handle, tf's getRPY, pcl::getTransformation and Eigen's Affine3f.
 * The node's main() is renamed so the library has none; every line of the node's callbacks that runs here is the
 * reference's.  Messages go in through the public callbacks (ImuCallback, OdomCallback, ScanCallback); the published
 * cloud, and the state the node computed it from, come back out.
 *
 * The node keeps its per-scan state (the IMU table, the odometry messages it chose) in private members.  They are read
 * here, not changed: the node's header is included with `private` spelled `public`, after every other header it pulls
 * in, so that only the node's class is affected.
 */
#include <chrono>
#include <cmath>
#include <cstring>
#include <deque>
#include <iostream>
#include <mutex>
#include <vector>

#include <ros/ros.h>
#include <sensor_msgs/LaserScan.h>
#include <sensor_msgs/PointCloud2.h>
#include <sensor_msgs/Imu.h>
#include <nav_msgs/Odometry.h>
#include <tf/LinearMath/Quaternion.h>
#include <tf/transform_datatypes.h>
#include <pcl_ros/point_cloud.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include <pcl/common/common.h>
#include <pcl/common/transforms.h>

#define private public
#include <lesson5/lidar_undistortion.h>
#undef private

#define main lesson5_lidar_undistortion_main
#include "lesson5/src/lidar_undistortion.cc"
#undef main

namespace {

LidarUndistortion *node = nullptr;

/* the state one published cloud was computed from, captured inside publish() (before ResetParameters) */
struct Published {
  uint32_t sec, nsec;          /* header stamp of the corrected scan */
  double scan_start, scan_end; /* current_scan_time_start_ / _end_ */
  int32_t imu_last;            /* current_imu_index_ */
  double odom_start_time, odom_end_time;
  double start_pose[6], end_pose[6]; /* x, y, z, roll, pitch, yaw of start_odom_msg_ / end_odom_msg_ (getRPY) */
  float odom_incre[3];
  std::vector<float> xyz;
  std::vector<double> imu_time, rot_x, rot_y, rot_z;
} last;

void pose_of(const nav_msgs::Odometry &m, double out[6]) {
  out[0] = m.pose.pose.position.x;
  out[1] = m.pose.pose.position.y;
  out[2] = m.pose.pose.position.z;
  tf::Quaternion q;
  tf::quaternionMsgToTF(m.pose.pose.orientation, q);
  tf::Matrix3x3(q).getRPY(out[3], out[4], out[5]);  // the node's own call sequence (:308-309)
}

void capture() {
  const LidarUndistortion &n = *node;
  last.sec = n.current_laserscan_header_.stamp.sec;
  last.nsec = n.current_laserscan_header_.stamp.nsec;
  last.scan_start = n.current_scan_time_start_;
  last.scan_end = n.current_scan_time_end_;
  last.imu_last = n.current_imu_index_;
  last.odom_start_time = last.odom_end_time = 0.0;  // without use_odometry the node never sets them
  std::memset(last.start_pose, 0, sizeof last.start_pose);
  std::memset(last.end_pose, 0, sizeof last.end_pose);
  if (n.use_odom_) {
    last.odom_start_time = n.start_odom_time_;
    last.odom_end_time = n.end_odom_time_;
    pose_of(n.start_odom_msg_, last.start_pose);
    pose_of(n.end_odom_msg_, last.end_pose);
  }
  last.odom_incre[0] = n.odom_incre_x_;
  last.odom_incre[1] = n.odom_incre_y_;
  last.odom_incre[2] = n.odom_incre_z_;
  const auto &cloud = ros::shim::last_published<pcl::PointCloud<pcl::PointXYZ>>();
  last.xyz.clear();
  for (const auto &p : cloud.points) {
    last.xyz.push_back(p.x);
    last.xyz.push_back(p.y);
    last.xyz.push_back(p.z);
  }
  last.imu_time = n.imu_time_;
  last.rot_x = n.imu_rot_x_;
  last.rot_y = n.imu_rot_y_;
  last.rot_z = n.imu_rot_z_;
}

std_msgs::Header header(uint32_t sec, uint32_t nsec) {
  std_msgs::Header h;
  h.stamp.sec = sec;
  h.stamp.nsec = nsec;
  return h;
}

}  // namespace

extern "C" {

/* a fresh node with the parameters use_imu / use_odometry */
void ref_deskew_new(int use_imu, int use_odom) {
  delete node;
  ros::shim::params()["use_imu"] = use_imu;
  ros::shim::params()["use_odometry"] = use_odom;
  node = new LidarUndistortion();
  ros::shim::publish_hook() = capture;
}

void ref_deskew_imu(uint32_t sec, uint32_t nsec, double wx, double wy, double wz) {
  auto m = std::make_shared<sensor_msgs::Imu>();
  m->header = header(sec, nsec);
  m->angular_velocity.x = wx;
  m->angular_velocity.y = wy;
  m->angular_velocity.z = wz;
  m->orientation.w = 1.0;
  sensor_msgs::Imu::ConstPtr c = m;
  node->ImuCallback(c);
}

/* position and orientation quaternion (x, y, z, w) */
void ref_deskew_odom(uint32_t sec, uint32_t nsec, const double pos[3], const double quat[4]) {
  auto m = std::make_shared<nav_msgs::Odometry>();
  m->header = header(sec, nsec);
  m->pose.pose.position.x = pos[0];
  m->pose.pose.position.y = pos[1];
  m->pose.pose.position.z = pos[2];
  m->pose.pose.orientation.x = quat[0];
  m->pose.pose.orientation.y = quat[1];
  m->pose.pose.orientation.z = quat[2];
  m->pose.pose.orientation.w = quat[3];
  nav_msgs::Odometry::ConstPtr c = m;
  node->OdomCallback(c);
}

/* ScanCallback on one LaserScan; fields[5] = angle_min, angle_increment, time_increment, range_min, range_max.
 * Returns 1 when the node published a cloud (of the scan before this one), 0 when it did not. */
int ref_deskew_scan(uint32_t sec, uint32_t nsec, const float fields[5], int n, const float *ranges) {
  auto m = std::make_shared<sensor_msgs::LaserScan>();
  m->header = header(sec, nsec);
  m->angle_min = fields[0];
  m->angle_increment = fields[1];
  m->angle_max = fields[0] + (n - 1) * fields[1];
  m->time_increment = fields[2];
  m->range_min = fields[3];
  m->range_max = fields[4];
  m->ranges.assign(ranges, ranges + n);
  sensor_msgs::LaserScan::ConstPtr c = m;
  const unsigned long before = ros::shim::publish_count();
  node->ScanCallback(c);
  return ros::shim::publish_count() != before;
}

/* the last published cloud: stamp[2] (sec, nsec), times[4] = scan start, scan end, odometry start, odometry end,
 * poses[12] = start and end pose, incre[3], xyz[n][3]; imu tables [cap] (cap <= 2000).  Returns imu_last. */
int ref_deskew_published(uint32_t *stamp, double *times, double *poses, float *incre, int n, float *xyz, int cap,
                         double *imu_time, double *rx, double *ry, double *rz) {
  stamp[0] = last.sec;
  stamp[1] = last.nsec;
  times[0] = last.scan_start;
  times[1] = last.scan_end;
  times[2] = last.odom_start_time;
  times[3] = last.odom_end_time;
  std::memcpy(poses, last.start_pose, sizeof last.start_pose);
  std::memcpy(poses + 6, last.end_pose, sizeof last.end_pose);
  std::memcpy(incre, last.odom_incre, sizeof last.odom_incre);
  std::memset(xyz, 0, sizeof(float) * 3 * n);
  std::memcpy(xyz, last.xyz.data(), sizeof(float) * std::min<size_t>(3 * (size_t)n, last.xyz.size()));
  for (int i = 0; i < cap && i < (int)last.imu_time.size(); i++) {
    imu_time[i] = last.imu_time[i];
    rx[i] = last.rot_x[i];
    ry[i] = last.rot_y[i];
    rz[i] = last.rot_z[i];
  }
  return last.imu_last;
}

}  // extern "C"
