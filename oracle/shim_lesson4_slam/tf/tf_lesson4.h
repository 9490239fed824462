// TEST INFRASTRUCTURE, NOT tf — the tf (ROS 1) surface lesson4's hector_slam.cc uses, for compiling the node unmodified
// (oracle/ref_lesson4_slam.cpp), on top of lesson6's tf stand-in (oracle/shim_lesson6/tf/tf_core.h: LinearMath, the
// listener that answers base_link <- laser from the mount a driver sets).  Three of its types gain what this node needs:
//   StampedTransform      a default constructor (the node holds one as a member)
//   TransformListener     waitForTransform / lookupTransform (the constructor's lookup of the mount)
//   TransformBroadcaster  sendTransform hands every transform to a hook a driver sets
// They are derived from lesson6's types, which are included here under other names, so lesson6's build is unchanged.
// poseMsgToTF is tf's: Transform(Quaternion(orientation), Vector3(position)).
#pragma once

#include <functional>
#include <string>

#include "ros/ros.h"

#define StampedTransform StampedTransformBase
#define TransformListener TransformListenerBase
#define TransformBroadcaster TransformBroadcasterBase
#include "tf/tf_core.h"
#undef StampedTransform
#undef TransformListener
#undef TransformBroadcaster

#include "../../shim/tf/transform_datatypes.h"  // quaternionMsgToTF (lesson5's)

namespace tf {

struct StampedTransform : StampedTransformBase {
  StampedTransform() : StampedTransformBase(Transform(), ros::Time(), "", "") {}
  StampedTransform(const Transform &t, const ros::Time &ts, const std::string &frame, const std::string &child)
      : StampedTransformBase(t, ts, frame, child) {}
};

class TransformListener : public TransformListenerBase {
 public:
  bool waitForTransform(const std::string &target, const std::string &source, const ros::Time &, const ros::Duration &) const {
    try {
      lookup(target, source);
      return true;
    } catch (const TransformException &) {
      return false;
    }
  }
  void lookupTransform(const std::string &target, const std::string &source, const ros::Time &t, StampedTransform &out) const {
    out = StampedTransform(lookup(target, source), t, target, source);
  }
};

namespace shim {
// called with every transform a broadcaster sends
inline std::function<void(const StampedTransform &)> &on_send_transform() {
  static std::function<void(const StampedTransform &)> f;
  return f;
}
}  // namespace shim

struct TransformBroadcaster {
  void sendTransform(const StampedTransform &t) {
    if (shim::on_send_transform()) shim::on_send_transform()(t);
  }
};

inline void poseMsgToTF(const geometry_msgs::Pose &msg, Transform &bt) {
  bt = Transform(Quaternion(msg.orientation.x, msg.orientation.y, msg.orientation.z, msg.orientation.w),
                 Vector3(msg.position.x, msg.position.y, msg.position.z));
}

}  // namespace tf
