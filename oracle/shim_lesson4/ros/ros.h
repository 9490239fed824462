// TEST INFRASTRUCTURE — the part of roscpp that lesson4's make-map nodes (src/gmapping/gmapping.cc,
// src/hector_mapping/hector_mapping.cc) touch, so that the unmodified nodes compile and their callbacks can be called
// directly (oracle/ref_lesson4_gmapping.cpp, oracle/ref_lesson4_hector.cpp).  It takes the place of oracle/shim/ros/ros.h
// for those builds (this directory comes first on their include path): the nodes also need a private NodeHandle("~"),
// getParam into double and float members, ros::Time(sec, nsec) and ros::Time::now().  There is no master, no topic and
// no spinning: subscribe() records nothing, and publish() keeps the last message so the driver can read it back.
#pragma once

// real ROS headers pull these in transitively; the Hector map headers use UINT_MAX without including <climits>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <map>
#include <memory>
#include <string>

#include "sensor_msgs/LaserScan.h"

#define ROS_INFO_STREAM(args) \
  do {                        \
  } while (0)

namespace ros {

inline void init(int &, char **, const std::string &) {}
inline void spin() {}

struct Subscriber {};

struct Time {
  using Stamp = decltype(std_msgs::Header::stamp);  // a message header's stamp
  uint32_t sec = 0, nsec = 0;
  Time() = default;
  Time(uint32_t s, uint32_t ns) : sec(s), nsec(ns) {}
  Time(const Stamp &s) : sec(s.sec), nsec(s.nsec) {}
  operator Stamp() const {
    Stamp s;
    s.sec = sec;
    s.nsec = nsec;
    return s;
  }
  static Time now() { return Time(); }
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
// what NodeHandle::getParam reads: the driver sets a value by its name (without the node handle's namespace)
inline std::map<std::string, double> &params() {
  static std::map<std::string, double> p;
  return p;
}
}  // namespace shim

struct Publisher {
  template <class M>
  void publish(const M &m) const {
    shim::last_published<M>() = m;
    ++shim::publish_count();
  }
};

struct NodeHandle {
  NodeHandle() = default;
  explicit NodeHandle(const std::string &) {}
  template <class T, class A>
  Subscriber subscribe(const std::string &, uint32_t, void (T::*)(A), T *) { return Subscriber(); }
  // false (and `value` untouched) when the driver has not set the parameter; a set value is converted to T, as the
  // parameter server's double is converted to a float member
  template <class T>
  bool getParam(const std::string &name, T &value) const {
    const auto it = shim::params().find(name);
    if (it == shim::params().end()) return false;
    value = static_cast<T>(it->second);
    return true;
  }
  template <class M>
  Publisher advertise(const std::string &, uint32_t, bool = false) { return Publisher(); }
};

}  // namespace ros
