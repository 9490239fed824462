// TEST INFRASTRUCTURE — the part of roscpp that the unmodified nodes touch (lesson1's feature_detection.cc, lesson3's
// plicp_odometry.cc, lesson4's gmapping.cc and hector_mapping.cc, lesson5's lidar_undistortion.cc, lesson6's
// karto_slam.cc), so that they compile and their callbacks can be called directly (oracle/ref_lesson*.cpp).  There is
// no master, no topic and no spinning: subscribe() records nothing, publish() keeps the last message, counts it and
// calls the hooks a driver sets, and ros::ok() is false, so a node's transform-publish loop returns at once.
#pragma once

// real ROS headers pull these in transitively; the nodes call std::isfinite and std::sort without including them, and
// the Hector map headers use UINT_MAX without including <climits>.  No <math.h>: which cos / sin a node's unqualified
// calls bind to depends on it (DESIGN.md §7 (1)).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <string>

#include "sensor_msgs/LaserScan.h"

#define ROS_INFO(...) \
  do {                \
  } while (0)
#define ROS_INFO_STREAM(args) \
  do {                        \
  } while (0)
#define ROS_WARN(...) \
  do {                \
  } while (0)
#define ROS_DEBUG(...) \
  do {                 \
  } while (0)
#define ROS_ERROR(...) \
  do {                 \
  } while (0)

namespace ros {

inline void init(int &, char **, const std::string &) {}
inline void spin() {}
inline void waitForShutdown() {}
inline bool ok() { return false; }

// ros::Duration / ros::Time (roscpp_core rostime): a difference of two times is the (sec, nsec) differences, normalised
// so that 0 <= nsec < 1e9 (normalizeSecNSecSigned); fromSec takes floor(d) seconds and round((d - sec) * 1e9)
// nanoseconds, rolling a whole second over; a Duration compares by (sec, nsec); toSec() = sec + 1e-9 * nsec
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
  explicit Duration(double d) { fromSec(d); }
  Duration &fromSec(double d) {
    sec = (int32_t)(int64_t)std::floor(d);
    nsec = (int32_t)std::round((d - sec) * 1e9);
    int32_t rollover = nsec / 1000000000;
    sec += rollover;
    nsec %= 1000000000;
    return *this;
  }
  double toSec() const { return (double)sec + 1e-9 * (double)nsec; }
  bool operator>(const Duration &r) const { return sec > r.sec || (sec == r.sec && nsec > r.nsec); }
  bool sleep() const { return true; }
};

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
  Duration operator-(const Time &rhs) const { return Duration((int32_t)sec - (int32_t)rhs.sec, (int32_t)nsec - (int32_t)rhs.nsec); }
  Time operator+(const Duration &d) const {
    int64_t s = (int64_t)sec + d.sec, ns = (int64_t)nsec + d.nsec;
    s += ns / 1000000000LL;
    return Time((uint32_t)s, (uint32_t)(ns % 1000000000LL));
  }
};

// a header stamp minus a ros::Time, as roscpp's message stamps are ros::Time
inline Duration operator-(const Time::Stamp &a, const Time &b) { return Time(a) - b; }

struct Rate {
  explicit Rate(double) {}
  bool sleep() { return true; }
};

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
// called with every message of type M a publisher sends
template <class M>
std::function<void(const M &)> &on_publish() {
  static std::function<void(const M &)> f;
  return f;
}
// what NodeHandle::param / getParam read: the driver sets a value by its name (without the node handle's namespace);
// string parameters come from their own map, empty unless a driver sets one
inline std::map<std::string, double> &params() {
  static std::map<std::string, double> p;
  return p;
}
inline std::map<std::string, std::string> &string_params() {
  static std::map<std::string, std::string> p;
  return p;
}
}  // namespace shim

struct Publisher {
  template <class M>
  void publish(const M &m) const {
    shim::last_published<M>() = m;
    published(m);
  }
  // a message held by pointer is copied when it is published, as serialisation would copy it
  template <class M>
  void publish(const std::shared_ptr<M> &m) const {
    shim::last_published<M>() = *m;
    published(*m);
  }
  template <class M>
  static void published(const M &m) {
    ++shim::publish_count();
    if (shim::on_publish<M>()) shim::on_publish<M>()(m);
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
  // false (and `value` untouched) when the driver has not set the parameter; a set value is converted to T, as the
  // parameter server's double is converted to a float member
  template <class T>
  bool getParam(const std::string &name, T &value) const {
    const auto it = shim::params().find(name);
    if (it == shim::params().end()) return false;
    value = static_cast<T>(it->second);
    return true;
  }
  bool getParam(const std::string &name, std::string &value) const {
    const auto it = shim::string_params().find(name);
    if (it == shim::string_params().end()) return false;
    value = it->second;
    return true;
  }
  template <class T>
  bool param(const std::string &name, T &value, const T &fallback) const {
    if (getParam(name, value)) return true;
    value = fallback;
    return false;
  }
  // the node passes `this` as the third argument, which converts to advertise()'s `bool latch`
  template <class M>
  Publisher advertise(const std::string &, uint32_t, bool = false) { return Publisher(); }
};

}  // namespace ros
