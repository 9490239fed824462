// TEST INFRASTRUCTURE, NOT PCL — pcl::PointCloud and pcl::PCLHeader with the members lesson5's lidar_undistortion.cc
// touches (oracle/ref_lesson5.cpp).
#pragma once

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace pcl {
struct PCLHeader {
  uint32_t seq = 0;
  uint64_t stamp = 0;  // microseconds, as pcl_conversions stores a ROS stamp
  std::string frame_id;
};

template <class PointT>
struct PointCloud {
  PCLHeader header;
  std::vector<PointT> points;
  uint32_t width = 0, height = 0;
  bool is_dense = true;
  typedef std::shared_ptr<PointCloud> Ptr;
  typedef std::shared_ptr<const PointCloud> ConstPtr;
};
}  // namespace pcl
