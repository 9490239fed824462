// TEST INFRASTRUCTURE — the nav_msgs/GetMap service type (its response holds the map) for lesson6's karto_slam.cc.
#pragma once

#include "nav_msgs/OccupancyGrid.h"

namespace nav_msgs {
struct GetMap {
  struct Request {};
  struct Response {
    OccupancyGrid map;
  };
};
}  // namespace nav_msgs
