/*
 * mini_eigen.h — TEST INFRASTRUCTURE, NOT PRODUCT CODE, and NOT Eigen.
 *
 * Eigen is absent from this image and cannot be fetched, and every lesson4 Hector header includes <Eigen/...>.
 * This is the smallest stand-in for the fixed-size types those headers use (Vector2f/3f/4f/2i, Matrix3f,
 * Matrix<float,3,7>, Affine2f/3f, Translation2f/3f, Rotation2Df, AlignedScaling2f/3f) so that the UNMODIFIED
 * reference headers compile where they lie under the reference checkout (oracle/ref_hector.cpp); lesson5's
 * lidar_undistortion.cc uses Affine3f as well (oracle/ref_lesson5.cpp).  All the SLAM logic
 * that runs is then the reference's own; only these linear-algebra primitives are ours.  They mirror Eigen 3.3's
 * fixed-size behaviour as follows (scalar float, no vectorisation for these sizes, no FMA contraction in a build
 * without -march):
 *   Matrix(float, float) into an int vector         -> static_cast<int>, truncation toward zero
 *   .cast<int>()                                    -> static_cast<int> per coefficient
 *   A * v (fixed-size product)                      -> coeff(i) = redux(a(i,k)*v(k)): two terms p0 + p1, three terms p0 + (p1 + p2)
 *   Transform * v  (Affine mode)                    -> translation + linear*v  (same bits as linear*v + translation)
 *   Translation * Rotation2D                        -> linear = [[c,-s],[s,c]] with c = cosf(a), s = sinf(a); translation = t
 *   AlignedScaling * Translation                    -> linear = diag(s); translation = diag(s)*t
 *   Transform::inverse() (Affine)                   -> L' = L.inverse(); t' = -(L' * t)
 *   Affine3f * Affine3f                             -> L = L1 * L2; t = L1 * t2 + t1
 *   2x2 / 3x3 inverse                               -> cofactor / determinant forms, multiplied by 1/det
 * Re-verify against a real Eigen build whenever one is available.
 */
#pragma once
#include <cmath>
#include <cstddef>
#include <ostream>

#define EIGEN_MAKE_ALIGNED_OPERATOR_NEW

namespace Eigen {

template <typename T, int R, int C>
struct Matrix;

/* Eigen's unrolled scalar reduction (redux_novec_unroller): halves the range recursively, so three terms sum as
 * a0 + (a1 + a2).  Fixed-size coefficient products and .sum()/.dot()/.squaredNorm() all go through it. */
template <typename T>
inline T redux_sum(const T *a, int start, int len) {
  if (len == 1) return a[start];
  int half = len / 2;
  return redux_sum(a, start, half) + redux_sum(a, start + half, len - half);
}

template <typename T, int R, int C, int BR, int BC>
struct BlockRef {
  Matrix<T, R, C> &m;
  int r0, c0;
  BlockRef &operator=(const Matrix<T, BR, BC> &o) {
    for (int j = 0; j < BC; ++j)
      for (int i = 0; i < BR; ++i) m(r0 + i, c0 + j) = o(i, j);
    return *this;
  }
  operator Matrix<T, BR, BC>() const {
    Matrix<T, BR, BC> o;
    for (int j = 0; j < BC; ++j)
      for (int i = 0; i < BR; ++i) o(i, j) = m(r0 + i, c0 + j);
    return o;
  }
  Matrix<T, BR, BC> operator*(T s) const { return Matrix<T, BR, BC>(*this) * s; }
  Matrix<T, BR, BC> operator-(const Matrix<T, BR, BC> &o) const { return Matrix<T, BR, BC>(*this) - o; }
};

template <typename T, int R, int C>
struct ArrayView { /* .array(): coefficient-wise view */
  Matrix<T, R, C> &v;
  ArrayView &operator+=(T s) {
    for (int i = 0; i < R * C; ++i) v.d[i] += s;
    return *this;
  }
  ArrayView &operator-=(T s) {
    for (int i = 0; i < R * C; ++i) v.d[i] -= s;
    return *this;
  }
  Matrix<T, R, C> operator-(T s) const {
    Matrix<T, R, C> o;
    for (int i = 0; i < R * C; ++i) o.d[i] = v.d[i] - s;
    return o;
  }
  Matrix<T, R, C> operator+(T s) const {
    Matrix<T, R, C> o;
    for (int i = 0; i < R * C; ++i) o.d[i] = v.d[i] + s;
    return o;
  }
};

template <typename T, int R, int C>
struct Matrix {
  T d[R * C]; /* column-major, Eigen's default */
  typedef T Scalar;

  Matrix() {}
  template <typename A, typename B>
  Matrix(const A &x, const B &y) {
    static_assert(R * C == 2, "2-coefficient constructor");
    d[0] = static_cast<T>(x);
    d[1] = static_cast<T>(y);
  }
  template <typename A, typename B, typename D>
  Matrix(const A &x, const B &y, const D &z) {
    static_assert(R * C == 3, "3-coefficient constructor");
    d[0] = static_cast<T>(x);
    d[1] = static_cast<T>(y);
    d[2] = static_cast<T>(z);
  }
  template <typename A, typename B, typename D, typename E>
  Matrix(const A &x, const B &y, const D &z, const E &w) {
    static_assert(R * C == 4, "4-coefficient constructor");
    d[0] = static_cast<T>(x);
    d[1] = static_cast<T>(y);
    d[2] = static_cast<T>(z);
    d[3] = static_cast<T>(w);
  }

  static Matrix Zero() {
    Matrix m;
    for (int i = 0; i < R * C; ++i) m.d[i] = T(0);
    return m;
  }
  static Matrix Identity() {
    Matrix m = Zero();
    for (int i = 0; i < (R < C ? R : C); ++i) m(i, i) = T(1);
    return m;
  }

  T &operator()(int i, int j) { return d[j * R + i]; }
  const T &operator()(int i, int j) const { return d[j * R + i]; }
  T &operator()(int i) { return d[i]; }
  const T &operator()(int i) const { return d[i]; }
  T &operator[](int i) { return d[i]; }
  const T &operator[](int i) const { return d[i]; }
  T &x() { return d[0]; }
  const T &x() const { return d[0]; }
  T &y() { return d[1]; }
  const T &y() const { return d[1]; }
  T &z() { return d[2]; }
  const T &z() const { return d[2]; }
  int rows() const { return R; }
  int cols() const { return C; }

  template <int N>
  Matrix<T, N, 1> head() const {
    static_assert(C == 1 && N <= R, "head<N> of a column vector");
    Matrix<T, N, 1> o;
    for (int i = 0; i < N; ++i) o.d[i] = d[i];
    return o;
  }
  template <typename U>
  Matrix<U, R, C> cast() const {
    Matrix<U, R, C> o;
    for (int i = 0; i < R * C; ++i) o.d[i] = static_cast<U>(d[i]);
    return o;
  }
  ArrayView<T, R, C> array() { return ArrayView<T, R, C>{*this}; }
  ArrayView<T, R, C> array() const { return ArrayView<T, R, C>{const_cast<Matrix &>(*this)}; }
  T sum() const { return redux_sum(d, 0, R * C); }
  template <int BR, int BC>
  BlockRef<T, R, C, BR, BC> block(int r0, int c0) {
    return BlockRef<T, R, C, BR, BC>{*this, r0, c0};
  }
  Matrix<T, C, R> transpose() const {
    Matrix<T, C, R> o;
    for (int j = 0; j < C; ++j)
      for (int i = 0; i < R; ++i) o(j, i) = (*this)(i, j);
    return o;
  }
  T squaredNorm() const { return dot(*this); }
  T norm() const { return std::sqrt(squaredNorm()); }
  T dot(const Matrix &o) const {
    T p[R * C];
    for (int i = 0; i < R * C; ++i) p[i] = d[i] * o.d[i];
    return redux_sum(p, 0, R * C);
  }

  Matrix operator+(const Matrix &o) const {
    Matrix r;
    for (int i = 0; i < R * C; ++i) r.d[i] = d[i] + o.d[i];
    return r;
  }
  Matrix operator-(const Matrix &o) const {
    Matrix r;
    for (int i = 0; i < R * C; ++i) r.d[i] = d[i] - o.d[i];
    return r;
  }
  Matrix operator-() const {
    Matrix r;
    for (int i = 0; i < R * C; ++i) r.d[i] = -d[i];
    return r;
  }
  Matrix operator*(T s) const {
    Matrix r;
    for (int i = 0; i < R * C; ++i) r.d[i] = d[i] * s;
    return r;
  }
  Matrix operator/(T s) const {
    Matrix r;
    for (int i = 0; i < R * C; ++i) r.d[i] = d[i] / s;
    return r;
  }
  Matrix &operator+=(const Matrix &o) {
    for (int i = 0; i < R * C; ++i) d[i] += o.d[i];
    return *this;
  }
  Matrix &operator-=(const Matrix &o) {
    for (int i = 0; i < R * C; ++i) d[i] -= o.d[i];
    return *this;
  }
  Matrix &operator*=(T s) {
    for (int i = 0; i < R * C; ++i) d[i] *= s;
    return *this;
  }
  Matrix &operator/=(T s) {
    for (int i = 0; i < R * C; ++i) d[i] /= s;
    return *this;
  }
  template <int K>
  Matrix<T, R, K> operator*(const Matrix<T, C, K> &o) const {
    Matrix<T, R, K> r;
    for (int j = 0; j < K; ++j)
      for (int i = 0; i < R; ++i) {
        T p[C];
        for (int k = 0; k < C; ++k) p[k] = (*this)(i, k) * o(k, j);
        r(i, j) = redux_sum(p, 0, C);
      }
    return r;
  }
  bool operator==(const Matrix &o) const {
    for (int i = 0; i < R * C; ++i)
      if (!(d[i] == o.d[i])) return false;
    return true;
  }
  bool operator!=(const Matrix &o) const { return !(*this == o); }

  T determinant() const {
    static_assert(R == C && (R == 2 || R == 3), "determinant: 2x2 / 3x3 only");
    const Matrix &m = *this;
    if (R == 2) return m(0, 0) * m(1, 1) - m(1, 0) * m(0, 1);
    /* Eigen bruteforce_det3_helper summed over a = 0,1,2 */
    return (m(0, 0) * (m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2)) - m(1, 0) * (m(0, 1) * m(2, 2) - m(2, 1) * m(0, 2))) +
           m(2, 0) * (m(0, 1) * m(1, 2) - m(1, 1) * m(0, 2));
  }
  Matrix inverse() const {
    static_assert(R == C && (R == 2 || R == 3), "inverse: 2x2 / 3x3 only");
    const Matrix &m = *this;
    Matrix r;
    if (R == 2) { /* compute_inverse_size2_helper */
      T invdet = T(1) / determinant();
      r(0, 0) = m(1, 1) * invdet;
      r(1, 0) = -m(1, 0) * invdet;
      r(0, 1) = -m(0, 1) * invdet;
      r(1, 1) = m(0, 0) * invdet;
      return r;
    }
    /* compute_inverse_size3_helper: cofactors, det from the first cofactor column, result = cofactor^T * (1/det) */
    T cof[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        cof[i][j] = m(i1, j1) * m(i2, j2) - m(i1, j2) * m(i2, j1);
      }
    T det = cof[0][0] * m(0, 0) + (cof[1][0] * m(1, 0) + cof[2][0] * m(2, 0));
    T invdet = T(1) / det;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) r(i, j) = cof[j][i] * invdet;
    return r;
  }
};

template <typename T, int R, int C>
inline Matrix<T, R, C> operator*(T s, const Matrix<T, R, C> &m) {
  Matrix<T, R, C> r;
  for (int i = 0; i < R * C; ++i) r.d[i] = s * m.d[i];
  return r;
}

template <typename T, int R, int C>
inline std::ostream &operator<<(std::ostream &os, const Matrix<T, R, C> &m) {
  for (int i = 0; i < R; ++i) {
    for (int j = 0; j < C; ++j) os << (j ? " " : "") << m(i, j);
    if (i + 1 < R) os << "\n";
  }
  return os;
}

typedef Matrix<float, 2, 1> Vector2f;
typedef Matrix<float, 3, 1> Vector3f;
typedef Matrix<float, 4, 1> Vector4f;
typedef Matrix<int, 2, 1> Vector2i;
typedef Matrix<float, 2, 2> Matrix2f;
typedef Matrix<float, 3, 3> Matrix3f;

enum TransformTraits { Isometry = 0x1, Affine = 0x2, AffineCompact = 0x10 | Affine, Projective = 0x20 };

template <typename T, int Dim>
struct Translation {
  Matrix<T, Dim, 1> v;
  Translation() {}
  Translation(const T &x, const T &y) : v(x, y) {}
  Translation(const T &x, const T &y, const T &z) : v(x, y, z) {}
};

template <typename T>
struct Rotation2D {
  T a;
  explicit Rotation2D(const T &angle) : a(angle) {}
  Matrix<T, 2, 2> toRotationMatrix() const {
    T s = std::sin(a), c = std::cos(a);
    Matrix<T, 2, 2> m;
    m(0, 0) = c;
    m(0, 1) = -s;
    m(1, 0) = s;
    m(1, 1) = c;
    return m;
  }
};

template <typename T, int Dim>
struct DiagonalScaling {
  Matrix<T, Dim, 1> s;
  DiagonalScaling(const T &x, const T &y) : s(x, y) {}
  DiagonalScaling(const T &x, const T &y, const T &z) : s(x, y, z) {}
};

template <typename T, int Dim, int Mode = Affine>
struct Transform {
  Matrix<T, Dim, Dim> lin;
  Matrix<T, Dim, 1> tr;
  Transform() {}
  const Matrix<T, Dim, Dim> &linear() const { return lin; }
  const Matrix<T, Dim, 1> &translation() const { return tr; }
  Matrix<T, Dim, 1> operator*(const Matrix<T, Dim, 1> &p) const { return tr + lin * p; }
  Transform inverse() const {
    Transform r;
    r.lin = lin.inverse();
    r.tr = -(r.lin * tr);
    return r;
  }
};

/* the 3-D transform of GridMapBase::setMapTransformation (unused there), and lesson5's Affine3f (oracle/ref_lesson5.cpp):
 * coefficient (i, j) of the 4x4 matrix, and the product of two transforms as linear = L1 L2, translation = L1 t2 + t1,
 * each coefficient a three-term redux p0 + (p1 + p2), as csrc/lidar_undistortion.cu restates Eigen's product */
template <typename T, int Mode>
struct Transform<T, 3, Mode> {
  Matrix<T, 3, 3> lin;
  Matrix<T, 3, 1> tr;
  Transform() {}
  Matrix<T, 3, 1> operator*(const Matrix<T, 3, 1> &p) const { return tr + lin * p; }
  Transform operator*(const Transform &o) const {
    Transform r;
    r.lin = lin * o.lin;
    r.tr = lin * o.tr + tr;
    return r;
  }
  T operator()(int i, int j) const { return i == 3 ? T(j == 3 ? 1 : 0) : j == 3 ? tr[i] : lin(i, j); }
  Transform inverse() const {
    Transform r;
    r.lin = lin.inverse();
    r.tr = -(r.lin * tr);
    return r;
  }
};

template <typename T>
inline Transform<T, 2, Affine> operator*(const Translation<T, 2> &t, const Rotation2D<T> &r) {
  Transform<T, 2, Affine> o;
  o.lin = r.toRotationMatrix();
  o.tr = t.v;
  return o;
}

template <typename T, int Dim>
inline Transform<T, Dim, Affine> operator*(const DiagonalScaling<T, Dim> &s, const Translation<T, Dim> &t) {
  Transform<T, Dim, Affine> o;
  o.lin = Matrix<T, Dim, Dim>::Zero();
  for (int i = 0; i < Dim; ++i) {
    o.lin(i, i) = s.s[i];
    o.tr[i] = s.s[i] * t.v[i];
  }
  return o;
}

typedef Transform<float, 2, Affine> Affine2f;
typedef Transform<float, 3, Affine> Affine3f;
typedef Translation<float, 2> Translation2f;
typedef Translation<float, 3> Translation3f;
typedef Rotation2D<float> Rotation2Df;
typedef DiagonalScaling<float, 2> AlignedScaling2f;
typedef DiagonalScaling<float, 3> AlignedScaling3f;

} /* namespace Eigen */
