// TEST INFRASTRUCTURE, NOT PCL — pcl::PointXYZ (x, y, z, and the padding word PCL sets to 1) for compiling lesson5's
// lidar_undistortion.cc unmodified (oracle/ref_lesson5.cpp).
#pragma once

namespace pcl {
struct PointXYZ {
  float x = 0.0f, y = 0.0f, z = 0.0f, pad = 1.0f;
};
}  // namespace pcl
