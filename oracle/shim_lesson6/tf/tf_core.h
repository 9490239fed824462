// TEST INFRASTRUCTURE, NOT tf — the tf (ROS 1) types lesson6's karto_slam.cc uses, for compiling the node unmodified
// (oracle/ref_lesson6.cpp).  tf is not in the reference tree; its LinearMath is the tf2 stand-in
// (oracle/shim/tf2/LinearMath/Transform.h, under tf's names in oracle/shim/tf/LinearMath/: tf's Transform, Matrix3x3 and
// Quaternion share that arithmetic, operation by operation in double), with the few members tf adds:
// Vector3::setValue, Transform(Quaternion, Vector3), Stamped<T>, StampedTransform, createQuaternionFromRPY and getYaw
// (the yaw of Matrix3x3::getRPY).
// The listener answers every lookup from what the driver set: base_link <- laser is the mount, odom <- base_link the
// scan's odometry row (a row holding a NaN makes the lookup throw tf::TransformException).  Timing, interpolation and
// the transform tree of real tf are not modelled; the library restates exactly this arithmetic (DESIGN.md §7).
#pragma once

#include <cmath>
#include <stdexcept>
#include <string>

#include "ros/ros.h"
#include "tf/LinearMath/Matrix3x3.h"

namespace tf {

struct Vector3 : tf2::Vector3 {
  Vector3() = default;
  Vector3(double x, double y, double z) : tf2::Vector3(x, y, z) {}
  Vector3(const tf2::Vector3 &o) : tf2::Vector3(o) {}
  void setValue(double x, double y, double z) { v[0] = x; v[1] = y; v[2] = z; }
};
typedef Vector3 Point;

class Transform : public tf2::Transform {
 public:
  Transform() = default;
  Transform(const tf2::Transform &t) : tf2::Transform(t) {}
  Transform(const Quaternion &q, const Vector3 &c) {
    setRotation(q);
    setOrigin(c);
  }
  Transform inverse() const { return tf2::Transform::inverse(); }
  Transform operator*(const Transform &t) const { return tf2::Transform::operator*(t); }
  Vector3 operator*(const Vector3 &x) const { return (*this)(x); }
  Vector3 getOrigin() const { return tf2::Transform::getOrigin(); }
};
typedef Transform Pose;

template <class T>
struct Stamped : T {
  ros::Time stamp_;
  std::string frame_id_;
  Stamped() : frame_id_("NO_ID_STAMPED_DEFAULT_CONSTRUCTION") {}
  Stamped(const T &input, const ros::Time &timestamp, const std::string &frame_id)
      : T(input), stamp_(timestamp), frame_id_(frame_id) {}
  void setData(const T &input) { *static_cast<T *>(this) = input; }
};

struct StampedTransform : Transform {
  ros::Time stamp_;
  std::string frame_id_, child_frame_id_;
  StampedTransform(const Transform &t, const ros::Time &ts, const std::string &frame, const std::string &child)
      : Transform(t), stamp_(ts), frame_id_(frame), child_frame_id_(child) {}
};

inline Quaternion createQuaternionFromRPY(double roll, double pitch, double yaw) {
  Quaternion q;
  q.setRPY(roll, pitch, yaw);
  return q;
}

inline double getYaw(const Quaternion &q) {
  double roll, pitch, yaw;
  Matrix3x3(q).getRPY(roll, pitch, yaw);
  return yaw;
}

struct TransformException : std::runtime_error {
  explicit TransformException(const std::string &s) : std::runtime_error(s) {}
};

namespace shim {
// what the listener answers: the mount (base_link <- laser) and the current scan's odom <- base_link
struct Frames {
  Transform base_laser, odom_base;
  bool odom_ok = false;
  int odom_failures = 0;  // lookups of odom <- base_link that threw
};
inline Frames &frames() {
  static Frames f;
  return f;
}
}  // namespace shim

class TransformListener {
 public:
  // lookupTransform(target, source): every frame other than base_link and odom is the laser
  Transform lookup(const std::string &target, const std::string &source) const {
    shim::Frames &f = shim::frames();
    if (target == source) return Transform();
    if (target == "base_link" && source != "odom") return f.base_laser;
    if (source == "base_link" && target != "odom") return f.base_laser.inverse();
    if (target == "odom" && source == "base_link") {
      if (!f.odom_ok) {
        ++f.odom_failures;
        throw TransformException("odom <- base_link is not available at this stamp");
      }
      return f.odom_base;
    }
    throw TransformException("no transform " + target + " <- " + source);
  }
  // tf: stamped_out.setData(transform * stamped_in), stamped at the input's time in the target frame
  void transformPose(const std::string &target, const Stamped<Pose> &in, Stamped<Pose> &out) const {
    const Transform t = lookup(target, in.frame_id_);
    const ros::Time stamp = in.stamp_;
    out.setData(t * static_cast<const Transform &>(in));
    out.stamp_ = stamp;
    out.frame_id_ = target;
  }
  void transformPoint(const std::string &target, const Stamped<Point> &in, Stamped<Point> &out) const {
    const Transform t = lookup(target, in.frame_id_);
    const ros::Time stamp = in.stamp_;
    out.setData(t * static_cast<const Vector3 &>(in));
    out.stamp_ = stamp;
    out.frame_id_ = target;
  }
};

struct TransformBroadcaster {
  void sendTransform(const StampedTransform &) {}
};

}  // namespace tf
