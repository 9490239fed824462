// TEST INFRASTRUCTURE — tf::MessageFilter for compiling lesson6's karto_slam.cc unmodified: it queues nothing and calls
// nothing; the driver calls the node's laserCallback itself once the odometry for the scan's stamp is set.
#pragma once

#include <string>

#include "message_filters/subscriber.h"
#include "tf/tf_core.h"

namespace tf {
template <class M>
struct MessageFilter {
  MessageFilter(message_filters::Subscriber<M> &, TransformListener &, const std::string &, uint32_t) {}
  template <class F>
  void registerCallback(F) {}
};
}  // namespace tf
