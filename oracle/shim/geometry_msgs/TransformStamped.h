// TEST INFRASTRUCTURE — geometry_msgs Transform and TransformStamped with the fields of the ROS message definitions, for
// compiling lesson3's plicp_odometry.cc unmodified (oracle/ref_lesson3.cpp).
#pragma once

#include <string>

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace geometry_msgs {
struct Transform { Vector3 translation; Quaternion rotation; };
struct TransformStamped { std_msgs::Header header; std::string child_frame_id; Transform transform; };
}  // namespace geometry_msgs
