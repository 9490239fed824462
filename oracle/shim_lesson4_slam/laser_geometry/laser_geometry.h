// TEST INFRASTRUCTURE, NOT laser_geometry — LaserProjection::projectLaser in its sensor_msgs::PointCloud form, for
// compiling lesson4's hector_slam.cc unmodified (oracle/ref_lesson4_slam.cpp).  The package is not in the reference tree;
// this follows the rule DESIGN.md §7 states for it: beam i's unit vector is cos / sin(angle_min + (double)i *
// angle_increment) in double; a beam is kept iff range < range_cutoff (double; a negative cutoff means range_max) and
// range >= range_min (float); x = (float)((double)range * ux), likewise y, z = 0; kept beams stay in beam order.
#pragma once

#include <cmath>
#include <vector>

#include "sensor_msgs/LaserScan.h"

namespace geometry_msgs {
struct Point32 { float x = 0, y = 0, z = 0; };
}  // namespace geometry_msgs

namespace sensor_msgs {
struct PointCloud {
  std_msgs::Header header;
  std::vector<geometry_msgs::Point32> points;
};
}  // namespace sensor_msgs

namespace laser_geometry {
class LaserProjection {
 public:
  void projectLaser(const sensor_msgs::LaserScan &scan, sensor_msgs::PointCloud &cloud, double range_cutoff = -1.0) {
    const double cutoff = range_cutoff < 0.0 ? (double)scan.range_max : range_cutoff;
    cloud.header = scan.header;
    cloud.points.clear();
    for (size_t i = 0; i < scan.ranges.size(); i++) {
      const float r = scan.ranges[i];
      if (!((double)r < cutoff && r >= scan.range_min)) continue;
      const double a = (double)scan.angle_min + (double)i * (double)scan.angle_increment;
      geometry_msgs::Point32 p;
      p.x = (float)((double)r * std::cos(a));
      p.y = (float)((double)r * std::sin(a));
      p.z = 0.0f;
      cloud.points.push_back(p);
    }
  }
};
}  // namespace laser_geometry
