// TEST INFRASTRUCTURE — nav_msgs/OccupancyGrid with the fields of the ROS message definition (oracle/ref_lesson4_*.cpp).
// `data` is std::vector<int8_t>, as roscpp generates it: lesson4's hector_mapping.cc binds a reference to it.
#pragma once

#include <cstdint>
#include <memory>
#include <vector>

#include "nav_msgs/MapMetaData.h"
#include "sensor_msgs/LaserScan.h"

namespace nav_msgs {
struct OccupancyGrid {
  std_msgs::Header header;
  MapMetaData info;
  std::vector<int8_t> data;
  typedef std::shared_ptr<const OccupancyGrid> ConstPtr;
};
}  // namespace nav_msgs
