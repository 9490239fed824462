// TEST INFRASTRUCTURE — lesson5 includes sensor_msgs/PointCloud2.h but publishes a pcl::PointCloud (pcl_ros converts
// it on the wire); nothing of the message itself is used (oracle/ref_lesson5.cpp).
#pragma once

#include "sensor_msgs/LaserScan.h"
