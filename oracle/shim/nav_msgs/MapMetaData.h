// TEST INFRASTRUCTURE — nav_msgs/MapMetaData with the fields of the ROS message definition (oracle/ref_lesson4_*.cpp).
// `resolution` is float32 in the message: a node that computes its map width as (xmax - xmin) / info.resolution divides
// by the float-rounded cell size.
#pragma once

#include <cstdint>

#include "geometry_msgs/messages.h"
#include "sensor_msgs/LaserScan.h"

namespace nav_msgs {
struct MapMetaData {
  decltype(std_msgs::Header::stamp) map_load_time;
  float resolution = 0;
  uint32_t width = 0, height = 0;
  geometry_msgs::Pose origin;
};
}  // namespace nav_msgs
