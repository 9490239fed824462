// TEST INFRASTRUCTURE, NOT PCL — pcl::getTransformation and pcl::getTranslationAndEulerAngles for compiling lesson5's
// lidar_undistortion.cc unmodified (oracle/ref_lesson5.cpp).  PCL is not in the reference tree, so these restate
// PCL 1.8's published algorithms (common/impl/eigen.hpp) exactly as csrc/lidar_undistortion.cu and
// oracle/deskew_oracle.c restate them: float arithmetic, cos / sin of the float angles taken by the C library in double
// and rounded to float.  Together with the Affine3f product and inverse of shim/Eigen/mini_eigen.h they stay unpinned;
// every other line of the node that runs is the node's own.
#pragma once

#include <cmath>

#include <Eigen/Geometry>

namespace pcl {
inline Eigen::Affine3f getTransformation(float x, float y, float z, float roll, float pitch, float yaw) {
  const float A = (float)std::cos((double)yaw), B = (float)std::sin((double)yaw), C = (float)std::cos((double)pitch),
              D = (float)std::sin((double)pitch), E = (float)std::cos((double)roll), F = (float)std::sin((double)roll),
              DE = D * E, DF = D * F;
  Eigen::Affine3f t;
  t.lin(0, 0) = A * C; t.lin(0, 1) = A * DF - B * E; t.lin(0, 2) = B * F + A * DE; t.tr[0] = x;
  t.lin(1, 0) = B * C; t.lin(1, 1) = A * E + B * DF; t.lin(1, 2) = B * DE - A * F; t.tr[1] = y;
  t.lin(2, 0) = -D;    t.lin(2, 1) = C * F;          t.lin(2, 2) = C * E;          t.tr[2] = z;
  return t;
}

inline void getTranslationAndEulerAngles(const Eigen::Affine3f &t, float &x, float &y, float &z, float &roll, float &pitch,
                                         float &yaw) {
  x = t(0, 3);
  y = t(1, 3);
  z = t(2, 3);
  roll = std::atan2(t(2, 1), t(2, 2));
  pitch = std::asin(-t(2, 0));
  yaw = std::atan2(t(1, 0), t(0, 0));
}
}  // namespace pcl
