// TEST INFRASTRUCTURE, NOT tf — tf::Quaternion (tfScalar = double) for compiling lesson5's lidar_undistortion.cc
// unmodified (oracle/ref_lesson5.cpp).  tf is not in the reference tree; this restates only what the node uses.
#pragma once

#include <cmath>

namespace tf {
typedef double tfScalar;

class Quaternion {
 public:
  Quaternion() : x_(0), y_(0), z_(0), w_(1) {}
  Quaternion(tfScalar x, tfScalar y, tfScalar z, tfScalar w) : x_(x), y_(y), z_(z), w_(w) {}
  tfScalar x() const { return x_; }
  tfScalar y() const { return y_; }
  tfScalar z() const { return z_; }
  tfScalar w() const { return w_; }
  tfScalar length2() const { return x_ * x_ + y_ * y_ + z_ * z_ + w_ * w_; }

 private:
  tfScalar x_, y_, z_, w_;
};
}  // namespace tf
