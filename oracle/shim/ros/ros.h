// TEST INFRASTRUCTURE — the part of roscpp that lesson1's feature_detection.cc and lesson5's lidar_undistortion.cc touch,
// so that the unmodified nodes compile and their callbacks can be called directly (oracle/ref_lesson1.cpp,
// oracle/ref_lesson5.cpp).  There is no master, no topic and no
// spinning: subscribe() only records nothing, and publish() keeps the last message so the driver can read it back.
#pragma once

// real ROS headers pull these in transitively; the node calls std::isfinite and std::sort without including them
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <string>

#include "sensor_msgs/LaserScan.h"

#define ROS_INFO_STREAM(args) \
  do {                        \
  } while (0)
#define ROS_WARN(...) \
  do {                \
  } while (0)

namespace ros {

inline void init(int &, char **, const std::string &) {}
inline void spin() {}
inline void waitForShutdown() {}

struct Subscriber {};

struct AsyncSpinner {
  explicit AsyncSpinner(uint32_t) {}
  void start() {}
};

struct TransportHints {
  TransportHints &tcpNoDelay(bool = true) { return *this; }
};

namespace shim {
template <class M>
M &last_published() {
  static M m;
  return m;
}
// how many messages every publisher has sent; a driver compares it before and after a callback
inline unsigned long &publish_count() {
  static unsigned long n = 0;
  return n;
}
// called after every publish, while the node still holds the state the message was computed from
inline std::function<void()> &publish_hook() {
  static std::function<void()> f;
  return f;
}
// what NodeHandle::param reads: the driver sets a value by its name (without the node handle's namespace)
inline std::map<std::string, double> &params() {
  static std::map<std::string, double> p;
  return p;
}
}  // namespace shim

struct Publisher {
  template <class M>
  void publish(const M &m) const { shim::last_published<M>() = m; published(); }
  // a message held by pointer is copied when it is published, as serialisation would copy it
  template <class M>
  void publish(const std::shared_ptr<M> &m) const { shim::last_published<M>() = *m; published(); }
  static void published() {
    ++shim::publish_count();
    if (shim::publish_hook()) shim::publish_hook()();
  }
};

struct NodeHandle {
  NodeHandle() = default;
  explicit NodeHandle(const std::string &) {}
  template <class T, class A>
  Subscriber subscribe(const std::string &, uint32_t, void (T::*)(A), T *) { return Subscriber(); }
  template <class T, class A>
  Subscriber subscribe(const std::string &, uint32_t, void (T::*)(A), T *, const TransportHints &) { return Subscriber(); }
  template <class T>
  bool param(const std::string &name, T &value, const T &fallback) const {
    const auto it = shim::params().find(name);
    value = it == shim::params().end() ? fallback : static_cast<T>(it->second);
    return it != shim::params().end();
  }
  // the node passes `this` as the third argument, which converts to advertise()'s `bool latch`
  template <class M>
  Publisher advertise(const std::string &, uint32_t, bool = false) { return Publisher(); }
};

}  // namespace ros
