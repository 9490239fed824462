// TEST INFRASTRUCTURE — tf2's LinearMath (geometry2: tf2/LinearMath/{Vector3,Quaternion,Matrix3x3,Transform}.h) as far as
// the unmodified nodes use it: lesson3's plicp_odometry.cc (oracle/ref_lesson3.cpp), and through tf's names
// (tf/LinearMath/*.h, tf/tf_core.h) lesson5's lidar_undistortion.cc and lesson6's karto_slam.cc; tf's LinearMath is the
// same Bullet code.  Every operation is restated from geometry2's code, operation by operation in double (the drivers
// are built without FMA contraction): Matrix3x3 product through tdotx / tdoty / tdotz, Transform product (basis
// product, origin through dot3 + origin), inverse (transpose, transpose * -origin), setRotation / getRotation, getRPY
// and Quaternion::setRPY.  The library states the same arithmetic in csrc/ros_math.cuh; tests/ros_math_check.cpp holds
// the two equal.
//
// One deliberate difference: tf2 leaves a default-constructed Transform uninitialised, and the node reads one
// (plicp_odometry.cc:397, 423: corr_ch after a failed match).  Here the default constructor builds the IDENTITY, the
// rule the library follows (DESIGN.md §7): after a failed match only the scan-count rule can promote a key frame.
#pragma once

#include <cmath>

namespace tf2 {

typedef double tf2Scalar;

struct Vector3 {
  double v[3] = {0, 0, 0};
  Vector3() = default;
  Vector3(double x, double y, double z) : v{x, y, z} {}
  double x() const { return v[0]; }
  double y() const { return v[1]; }
  double z() const { return v[2]; }
  double getX() const { return v[0]; }
  double getY() const { return v[1]; }
  double getZ() const { return v[2]; }
  double dot(const Vector3 &o) const { return v[0] * o.v[0] + v[1] * o.v[1] + v[2] * o.v[2]; }
  Vector3 operator-() const { return Vector3(-v[0], -v[1], -v[2]); }
  Vector3 operator+(const Vector3 &o) const { return Vector3(v[0] + o.v[0], v[1] + o.v[1], v[2] + o.v[2]); }
  double operator[](int i) const { return v[i]; }
};

struct Quaternion {
  double q[4] = {0, 0, 0, 1};
  Quaternion() = default;
  Quaternion(double x, double y, double z, double w) : q{x, y, z, w} {}
  double x() const { return q[0]; }
  double y() const { return q[1]; }
  double z() const { return q[2]; }
  double w() const { return q[3]; }
  double getX() const { return q[0]; }
  double getY() const { return q[1]; }
  double getZ() const { return q[2]; }
  double getW() const { return q[3]; }
  void setValue(double x, double y, double z, double w) { q[0] = x; q[1] = y; q[2] = z; q[3] = w; }
  double length2() const { return q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]; }
  void setRPY(double roll, double pitch, double yaw) {
    double halfYaw = yaw * 0.5, halfPitch = pitch * 0.5, halfRoll = roll * 0.5;
    double cosYaw = std::cos(halfYaw), sinYaw = std::sin(halfYaw);
    double cosPitch = std::cos(halfPitch), sinPitch = std::sin(halfPitch);
    double cosRoll = std::cos(halfRoll), sinRoll = std::sin(halfRoll);
    setValue(sinRoll * cosPitch * cosYaw - cosRoll * sinPitch * sinYaw,
             cosRoll * sinPitch * cosYaw + sinRoll * cosPitch * sinYaw,
             cosRoll * cosPitch * sinYaw - sinRoll * sinPitch * cosYaw,
             cosRoll * cosPitch * cosYaw + sinRoll * sinPitch * sinYaw);
  }
};

struct Matrix3x3 {
  Vector3 el[3];
  Matrix3x3() = default;
  explicit Matrix3x3(const Quaternion &q) { setRotation(q); }
  Matrix3x3(double xx, double xy, double xz, double yx, double yy, double yz, double zx, double zy, double zz)
      : el{Vector3(xx, xy, xz), Vector3(yx, yy, yz), Vector3(zx, zy, zz)} {}
  const Vector3 &operator[](int i) const { return el[i]; }
  void setIdentity() { *this = Matrix3x3(1, 0, 0, 0, 1, 0, 0, 0, 1); }
  double tdotx(const Vector3 &v) const { return el[0].x() * v.x() + el[1].x() * v.y() + el[2].x() * v.z(); }
  double tdoty(const Vector3 &v) const { return el[0].y() * v.x() + el[1].y() * v.y() + el[2].y() * v.z(); }
  double tdotz(const Vector3 &v) const { return el[0].z() * v.x() + el[1].z() * v.y() + el[2].z() * v.z(); }
  Matrix3x3 transpose() const {
    return Matrix3x3(el[0].x(), el[1].x(), el[2].x(), el[0].y(), el[1].y(), el[2].y(), el[0].z(), el[1].z(), el[2].z());
  }
  void setRotation(const Quaternion &q) {
    double d = q.length2();
    double s = 2.0 / d;
    double xs = q.x() * s, ys = q.y() * s, zs = q.z() * s;
    double wx = q.w() * xs, wy = q.w() * ys, wz = q.w() * zs;
    double xx = q.x() * xs, xy = q.x() * ys, xz = q.x() * zs;
    double yy = q.y() * ys, yz = q.y() * zs, zz = q.z() * zs;
    *this = Matrix3x3(1.0 - (yy + zz), xy - wz, xz + wy, xy + wz, 1.0 - (xx + zz), yz - wx, xz - wy, yz + wx,
                      1.0 - (xx + yy));
  }
  void getRotation(Quaternion &q) const {
    double trace = el[0].x() + el[1].y() + el[2].z();
    double temp[4];
    if (trace > 0.0) {
      double s = std::sqrt(trace + 1.0);
      temp[3] = s * 0.5;
      s = 0.5 / s;
      temp[0] = (el[2].y() - el[1].z()) * s;
      temp[1] = (el[0].z() - el[2].x()) * s;
      temp[2] = (el[1].x() - el[0].y()) * s;
    } else {
      int i = el[0].x() < el[1].y() ? (el[1].y() < el[2].z() ? 2 : 1) : (el[0].x() < el[2].z() ? 2 : 0);
      int j = (i + 1) % 3;
      int k = (i + 2) % 3;
      double s = std::sqrt(el[i][i] - el[j][j] - el[k][k] + 1.0);
      temp[i] = s * 0.5;
      s = 0.5 / s;
      temp[3] = (el[k][j] - el[j][k]) * s;
      temp[j] = (el[j][i] + el[i][j]) * s;
      temp[k] = (el[k][i] + el[i][k]) * s;
    }
    q.setValue(temp[0], temp[1], temp[2], temp[3]);
  }
  // getEulerYPR, solution 1: R = Rz(yaw) Ry(pitch) Rx(roll); at the pitch singularity yaw is 0 and roll takes the
  // whole turn
  void getRPY(double &roll, double &pitch, double &yaw) const {
    if (std::fabs(el[2].x()) >= 1) {
      yaw = 0;
      const double delta = std::atan2(el[0].y(), el[0].z());
      if (el[2].x() > 0) {
        pitch = -M_PI / 2;
        roll = -yaw + std::atan2(-el[0].y(), -el[0].z());
      } else {
        pitch = M_PI / 2;
        roll = yaw + delta;
      }
      return;
    }
    pitch = -std::asin(el[2].x());
    const double c = std::cos(pitch);
    roll = std::atan2(el[2].y() / c, el[2].z() / c);
    yaw = std::atan2(el[1].x() / c, el[0].x() / c);
  }
};

inline Matrix3x3 operator*(const Matrix3x3 &m1, const Matrix3x3 &m2) {
  return Matrix3x3(m2.tdotx(m1[0]), m2.tdoty(m1[0]), m2.tdotz(m1[0]), m2.tdotx(m1[1]), m2.tdoty(m1[1]), m2.tdotz(m1[1]),
                   m2.tdotx(m1[2]), m2.tdoty(m1[2]), m2.tdotz(m1[2]));
}
inline Vector3 operator*(const Matrix3x3 &m, const Vector3 &v) { return Vector3(m[0].dot(v), m[1].dot(v), m[2].dot(v)); }

class Transform {
  Matrix3x3 m_basis;
  Vector3 m_origin;

 public:
  Transform() { setIdentity(); }  // tf2: uninitialised (see the header comment)
  Transform(const Matrix3x3 &b, const Vector3 &c) : m_basis(b), m_origin(c) {}
  // operator()(x) = x.dot3(basis rows) + origin
  Vector3 operator()(const Vector3 &x) const {
    return Vector3(x.dot(m_basis[0]), x.dot(m_basis[1]), x.dot(m_basis[2])) + m_origin;
  }
  Transform operator*(const Transform &t) const { return Transform(m_basis * t.m_basis, (*this)(t.m_origin)); }
  Transform inverse() const {
    Matrix3x3 inv = m_basis.transpose();
    return Transform(inv, inv * -m_origin);
  }
  void setIdentity() {
    m_basis.setIdentity();
    m_origin = Vector3(0, 0, 0);
  }
  const Vector3 &getOrigin() const { return m_origin; }
  void setOrigin(const Vector3 &o) { m_origin = o; }
  const Matrix3x3 &getBasis() const { return m_basis; }
  void setRotation(const Quaternion &q) { m_basis.setRotation(q); }
  Quaternion getRotation() const {
    Quaternion q;
    m_basis.getRotation(q);
    return q;
  }
};

}  // namespace tf2
