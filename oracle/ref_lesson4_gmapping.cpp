/*
 * ref_lesson4_gmapping.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson4 GMapping make-map node, reference/lesson4/src/gmapping/gmapping.cc,
 * #included where it lies (oracle/recipes.py builds it into _ref/liblesson4_ref.so).  ROS is absent; the stand-ins
 * under oracle/shim/ (the ROS core, LaserScan, OccupancyGrid, MapMetaData with a float32 resolution) provide the message types, the private node handle and its parameters.  The
 * node's main() is renamed so the library has none; every line of ScanCallback that runs here is the reference's.
 *
 * At its defaults the node's PublishMap writes past the end of map_.data (MAP_IDX(1599, x, y) for x, y < 1600 on a
 * vector of 1599 * 1599 bytes).  The driver reserves capacity behind the vector's end, fills it with SENTINEL, and
 * reports what the node wrote there, so the overrun lands in memory the driver owns.
 *
 * A ray that leaves the map's storage hits the node's assert(0) (map.h:186-191).  The driver checks every beam's end
 * cell with the node's own ScanMatcherMap before the callback and refuses the scan there instead of calling it.
 *
 * The node's header is included with `private` spelled `public`, after every other header it pulls in, so that only
 * the node's class is affected.
 */
#include <assert.h>
#include <math.h>

#include <chrono>
#include <cmath>
#include <cstring>
#include <iostream>
#include <memory>
#include <set>
#include <vector>

#include <ros/ros.h>
#include <sensor_msgs/LaserScan.h>
#include <nav_msgs/OccupancyGrid.h>
#include "lesson4/gmapping/grid/map.h"
#include "lesson4/gmapping/grid/gridlinetraversal.h"

#define private public
#include "lesson4/gmapping/gmapping.h"
#undef private

#define main lesson4_gmapping_main
#include "lesson4/src/gmapping/gmapping.cc"
#undef main

namespace {
gmapping::GMapping *node = nullptr;
size_t slack = 0;
constexpr int8_t SENTINEL = 0x55;  // never a published value (-1, 0, 100)
}  // namespace

extern "C" {

/* clear the parameter server; ref_l4_param sets one value; ref_l4_gmapping_new makes a fresh node with them */
void ref_l4_clear_params() { ros::shim::params().clear(); }
void ref_l4_param(const char *name, double value) { ros::shim::params()[name] = value; }

/* A fresh node.  out[2] = map_.info.width, height as InitParams computed them. */
void ref_l4_gmapping_new(int32_t out[2]) {
  delete node;
  std::cout.setstate(std::ios::failbit);  // the node prints its timing on every callback
  node = new gmapping::GMapping();
  std::vector<int8_t> &d = node->map_.data;
  // the largest index PublishMap forms is MAP_IDX(width, msx - 1, msy - 1) with the storage of its ScanMatcherMap
  gmapping::Point c((node->xmin_ + node->xmax_) / 2.0, (node->ymin_ + node->ymax_) / 2.0);
  gmapping::ScanMatcherMap m(c, node->xmin_, node->ymin_, node->xmax_, node->ymax_, node->resolution_);
  const size_t last = (size_t)node->map_.info.width * (m.getMapSizeY() - 1) + (m.getMapSizeX() - 1);
  slack = last + 1 > d.size() ? last + 1 - d.size() : 0;
  const size_t n = d.size();
  d.resize(n + slack, SENTINEL);  // capacity behind the end, owned by the vector
  d.resize(n);
  out[0] = (int32_t)node->map_.info.width;
  out[1] = (int32_t)node->map_.info.height;
}

/* ScanCallback on one LaserScan.  fields[4] = angle_min, angle_increment, range_min, range_max.  out [width*height] =
 * the published map_.data; overrun [overrun_cap] = the bytes behind the vector's end afterwards (SENTINEL where the node
 * wrote nothing), *n_overrun = how many of them the node wrote.  Returns 0, -1 when a beam's end cell lies outside the
 * storage (the node would assert; it is not called), -2 when nothing was published. */
int ref_l4_gmapping_scan(const float fields[4], int n, const float *ranges, int8_t *out, int8_t *overrun,
                         int overrun_cap, int32_t *n_overrun) {
  auto msg = std::make_shared<sensor_msgs::LaserScan>();
  msg->header.frame_id = "laser";
  msg->angle_min = fields[0];
  msg->angle_increment = fields[1];
  msg->angle_max = fields[0] + (n - 1) * fields[1];
  msg->range_min = fields[2];
  msg->range_max = fields[3];
  msg->ranges.assign(ranges, ranges + n);
  {
    // the beams' end cells, from the first scan's cache as CreateCache makes it (the driver calls the node with one
    // laser geometry) and ComputeMap's filter and world2map
    gmapping::Point c((node->xmin_ + node->xmax_) / 2.0, (node->ymin_ + node->ymax_) / 2.0);
    gmapping::ScanMatcherMap m(c, node->xmin_, node->ymin_, node->xmax_, node->ymax_, node->resolution_);
    const gmapping::IntPoint p0 = m.world2map(gmapping::Point(0, 0));  // the laser's cell starts every line
    const bool out0 = p0.x < 0 || p0.y < 0 || p0.x >= m.getMapSizeX() || p0.y >= m.getMapSizeY();
    for (int i = 0; i < n; i++) {
      double d = msg->ranges[i];
      if (d > node->max_range_ || d == 0.0 || !std::isfinite(d)) continue;
      if (d > node->max_use_range_) d = node->max_use_range_;
      const double angle = msg->angle_min + (unsigned)i * msg->angle_increment;
      gmapping::Point phit(0, 0);
      phit.x += d * cos(angle);
      phit.y += d * sin(angle);
      const gmapping::IntPoint p = m.world2map(phit);
      if (out0 || p.x < 0 || p.y < 0 || p.x >= m.getMapSizeX() || p.y >= m.getMapSizeY()) return -1;
    }
  }
  sensor_msgs::LaserScan::ConstPtr cmsg = msg;
  const unsigned long before = ros::shim::publish_count();
  node->ScanCallback(cmsg);
  if (ros::shim::publish_count() == before) return -2;
  const nav_msgs::OccupancyGrid &pub = ros::shim::last_published<nav_msgs::OccupancyGrid>();
  std::memcpy(out, pub.data.data(), pub.data.size());
  const int8_t *behind = node->map_.data.data() + node->map_.data.size();
  int32_t written = 0;
  for (size_t k = 0; k < slack; k++) {
    if ((int)k < overrun_cap) overrun[k] = behind[k];
    written += behind[k] != SENTINEL;
  }
  *n_overrun = written;
  return 0;
}

int ref_l4_gmapping_slack(void) { return (int)slack; }

}  // extern "C"
