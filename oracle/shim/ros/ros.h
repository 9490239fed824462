// TEST INFRASTRUCTURE — the part of roscpp that lesson1's feature_detection.cc touches, so that the unmodified node
// compiles and its ScanCallback can be called directly (oracle/ref_lesson1.cpp).  There is no master, no topic and no
// spinning: subscribe() only records nothing, and publish() keeps the last message so the driver can read it back.
#pragma once

// real ROS headers pull these in transitively; the node calls std::isfinite and std::sort without including them
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <string>

#include "sensor_msgs/LaserScan.h"

#define ROS_INFO_STREAM(args) \
  do {                        \
  } while (0)

namespace ros {

inline void init(int &, char **, const std::string &) {}
inline void spin() {}

struct Subscriber {};

namespace shim {
template <class M>
M &last_published() {
  static M m;
  return m;
}
}  // namespace shim

struct Publisher {
  template <class M>
  void publish(const M &m) const { shim::last_published<M>() = m; }
};

struct NodeHandle {
  NodeHandle() = default;
  explicit NodeHandle(const std::string &) {}
  template <class T, class A>
  Subscriber subscribe(const std::string &, uint32_t, void (T::*)(A), T *) { return Subscriber(); }
  // the node passes `this` as the third argument, which converts to advertise()'s `bool latch`
  template <class M>
  Publisher advertise(const std::string &, uint32_t, bool = false) { return Publisher(); }
};

}  // namespace ros
