// TEST INFRASTRUCTURE — visualization_msgs/Marker and MarkerArray with the fields lesson6's karto_slam.cc sets
// (publishGraphVisualization).
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "geometry_msgs/messages.h"
#include "ros/ros.h"

namespace visualization_msgs {
struct Marker {
  enum { ARROW = 0, CUBE = 1, SPHERE = 2, CYLINDER = 3, LINE_STRIP = 4 };
  enum { ADD = 0, MODIFY = 0, DELETE = 2 };
  std_msgs::Header header;
  std::string ns;
  int32_t id = 0, type = 0, action = 0;
  geometry_msgs::Pose pose;
  geometry_msgs::Vector3 scale;
  struct {
    float r = 0, g = 0, b = 0, a = 0;
  } color;
  ros::Duration lifetime;
  std::vector<geometry_msgs::Point> points;
};
struct MarkerArray {
  std::vector<Marker> markers;
};
}  // namespace visualization_msgs
