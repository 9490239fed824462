// TEST INFRASTRUCTURE — geometry_msgs Point, Vector3, Quaternion, Pose and the covariance-carrying wrappers, with the
// fields of the ROS message definitions, for compiling lesson5's lidar_undistortion.cc unmodified (oracle/ref_lesson5.cpp).
#pragma once

namespace geometry_msgs {
struct Point { double x = 0, y = 0, z = 0; };
struct Vector3 { double x = 0, y = 0, z = 0; };
struct Quaternion { double x = 0, y = 0, z = 0, w = 0; };
struct Pose { Point position; Quaternion orientation; };
struct PoseWithCovariance { Pose pose; double covariance[36] = {}; };
struct Twist { Vector3 linear, angular; };
struct TwistWithCovariance { Twist twist; double covariance[36] = {}; };
}  // namespace geometry_msgs
