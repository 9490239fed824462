// TEST INFRASTRUCTURE — message_filters::Subscriber for compiling lesson6's karto_slam.cc unmodified
// (oracle/ref_lesson6.cpp): it subscribes to nothing; the driver calls the node's laserCallback itself.
#pragma once

#include <string>

#include "ros/ros.h"

namespace message_filters {
template <class M>
struct Subscriber {
  Subscriber(ros::NodeHandle &, const std::string &, uint32_t) {}
};
}  // namespace message_filters
