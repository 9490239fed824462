// TEST INFRASTRUCTURE, NOT pcl_ros — lets a node publish a pcl::PointCloud (oracle/ref_lesson5.cpp).
#pragma once

#include "pcl/point_cloud.h"
#include "pcl/point_types.h"
#include "pcl_conversions/pcl_conversions.h"
