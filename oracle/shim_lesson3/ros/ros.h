// TEST INFRASTRUCTURE — the part of roscpp that lesson3's plicp_odometry.cc touches, so that the unmodified node compiles
// and its callback can be called directly (oracle/ref_lesson3.cpp).  It takes the place of oracle/shim/ros/ros.h for
// that one build (this directory comes first on its include path): the node also needs ros::Time / ros::Duration
// arithmetic, NodeHandle::getParam and string parameters.  There is no master, no topic and no spinning: subscribe()
// records nothing, and publish() keeps the last message so the driver can read it back.
#pragma once

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

struct Subscriber {};

// ros::Duration / ros::Time (roscpp_core rostime): a difference of two times is the (sec, nsec) differences, normalised
// so that 0 <= nsec < 1e9 (normalizeSecNSecSigned); toSec() = sec + 1e-9 * nsec
struct Duration {
  int32_t sec = 0, nsec = 0;
  Duration() = default;
  Duration(int32_t s, int32_t ns) {
    int64_t nsec_part = (int64_t)ns % 1000000000LL, sec_part = (int64_t)s + (int64_t)ns / 1000000000LL;
    if (nsec_part < 0) {
      nsec_part += 1000000000LL;
      --sec_part;
    }
    sec = (int32_t)sec_part;
    nsec = (int32_t)nsec_part;
  }
  explicit Duration(double) {}
  double toSec() const { return (double)sec + 1e-9 * (double)nsec; }
  bool sleep() const { return true; }
};

struct Time {
  using Stamp = decltype(std_msgs::Header::stamp);  // a message header's stamp
  uint32_t sec = 0, nsec = 0;
  Time() = default;
  Time(const Stamp &s) : sec(s.sec), nsec(s.nsec) {}
  operator Stamp() const {
    Stamp s;
    s.sec = sec;
    s.nsec = nsec;
    return s;
  }
  static Time now() { return Time(); }
  Duration operator-(const Time &rhs) const { return Duration((int32_t)sec - (int32_t)rhs.sec, (int32_t)nsec - (int32_t)rhs.nsec); }
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
// what NodeHandle::param / getParam read: the driver sets a value by its name (without the node handle's namespace)
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
  template <class T>
  bool param(const std::string &name, T &value, const T &fallback) const {
    const auto it = shim::params().find(name);
    value = it == shim::params().end() ? fallback : static_cast<T>(it->second);
    return it != shim::params().end();
  }
  // false (and `value` untouched) when the driver has not set the parameter
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

// string parameters (frame names) are never set by a driver: the fallback
template <>
inline bool NodeHandle::param<std::string>(const std::string &, std::string &value, const std::string &fallback) const {
  value = fallback;
  return false;
}

}  // namespace ros
