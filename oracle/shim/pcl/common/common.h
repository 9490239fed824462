// TEST INFRASTRUCTURE, NOT PCL — lesson5's lidar_undistortion.cc includes this header but uses nothing from it beyond
// what pcl/common/transforms.h provides (oracle/ref_lesson5.cpp).
#pragma once

#include "pcl/point_cloud.h"
#include "pcl/point_types.h"
