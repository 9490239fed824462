// TEST INFRASTRUCTURE — tf2_geometry_msgs toMsg / fromMsg (geometry2) as lesson3's plicp_odometry.cc calls them.
#pragma once

#include "geometry_msgs/TransformStamped.h"
#include "tf2/LinearMath/Transform.h"

namespace tf2 {
inline geometry_msgs::Quaternion toMsg(const Quaternion &in) {
  geometry_msgs::Quaternion out;
  out.x = in.getX(); out.y = in.getY(); out.z = in.getZ(); out.w = in.getW();
  return out;
}
inline geometry_msgs::Transform toMsg(const Transform &in) {
  geometry_msgs::Transform out;
  out.translation.x = in.getOrigin().getX();
  out.translation.y = in.getOrigin().getY();
  out.translation.z = in.getOrigin().getZ();
  out.rotation = toMsg(in.getRotation());
  return out;
}
inline geometry_msgs::Pose &toMsg(const Transform &in, geometry_msgs::Pose &out) {
  out.position.x = in.getOrigin().getX();
  out.position.y = in.getOrigin().getY();
  out.position.z = in.getOrigin().getZ();
  out.orientation = toMsg(in.getRotation());
  return out;
}
inline void fromMsg(const geometry_msgs::Transform &in, Transform &out) {
  out.setOrigin(Vector3(in.translation.x, in.translation.y, in.translation.z));
  out.setRotation(Quaternion(in.rotation.x, in.rotation.y, in.rotation.z, in.rotation.w));
}
}  // namespace tf2
