// TEST HELPER: the seeded sweep of inputs for csrc/ros_math.cuh, shared by ros_math_check.cpp (library, C restatements
// and node stand-ins on the host) and device_math_check.cu (the library's device build against its host build).  It
// reaches the branches node streams rarely take: getRotation with trace <= 0 (i = 0, 1, 2), getRPY at |m[2][0]| >= 1,
// tf2::getYaw at |sarg| >= 0.99999, negative nanosecond differences, the int32 wrap of seconds and the fromSec rollover.
// The sweep only draws inputs; the sink S decides what to compute from them:
//   s.quaternion(q)         a quaternion: setRotation, tf::getYaw, then the rotation checks
//   s.rpy(r, p, y)          roll / pitch / yaw: setRPY, then the quaternion checks
//   s.entries(m, o)         a transform entered directly: the rotation checks
//   s.chain(q, o, q2, o2, v) one chain of 12 products / inverses, step k combining with (q2[k], o2[k]), applied to v[k]
//   s.stamps(s1, n1, s0, n0) Time - Time, toSec
//   s.from_sec(d)           Duration::fromSec
//   s.from_sec_pair(d, d2)  Duration::fromSec of both and operator> both ways
#pragma once

#include <cmath>
#include <cstdint>
#include <random>

constexpr int ROS_MATH_CHAIN_STEPS = 12;

template <class S>
void ros_math_sweep(S &s) {
  std::mt19937_64 rng(20261016);
  std::uniform_real_distribution<double> u(-1.0, 1.0), scale(0.05, 20.0), big(-1e6, 1e6);
  std::uniform_int_distribution<uint32_t> any32;
  const double pi = 3.14159265358979323846;

  // quaternions: random unit and non-unit, zero, and each getRotation branch (w, then x, y or z largest), with ties
  const double crafted[][4] = {{0, 0, 0, 1},    {0, 0, 0, -1},  {0, 0, 0, 0},      {1, 0.1, 0.1, 0.05}, {0.1, 1, 0.1, 0.05},
                               {0.1, 0.1, 1, 0.05}, {1, 1, 0, 0}, {0, 1, 1, 0},     {1, 0, 1, 0},        {1, 1, 1, 0},
                               {1, 0, 0, 0},    {0, 1, 0, 0},   {0, 0, 1, 0},      {0, 1, 0, 1},        {0, 1, 0, -1},
                               {1, 1, -1, 1},   {1, 1, 1, -1},  {1e-300, 0, 0, 0}, {3, 4, 0, 0},        {-2, 0, 0, 1e-9}};
  for (const auto &q : crafted) s.quaternion(q);
  for (int n = 0; n < 20000; n++) {
    double q[4] = {u(rng), u(rng), u(rng), u(rng)};
    const double len = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double f = n % 2 ? scale(rng) : 1.0;
    for (double &x : q) x = x / len * f;
    if (n % 5 == 0) q[3] *= 1e-3;  // a small w: trace <= 0
    s.quaternion(q);
  }

  // roll / pitch / yaw, with pitch exactly +-90 degrees and just inside
  for (int n = 0; n < 5000; n++) s.rpy(pi * u(rng), 0.5 * pi * u(rng), pi * u(rng));
  for (double p : {pi / 2, -pi / 2}) {
    for (int k = 0; k < 40; k++) {
      const double inside = p - (p > 0 ? 1 : -1) * k * 1e-9;
      s.rpy(pi * u(rng), inside, pi * u(rng));
      s.rpy(0, inside, 0);
    }
  }
  // tf2::getYaw's sarg on both sides of +-0.99999: a pure pitch a has sarg = sin(a)
  const double edge = std::asin(0.99999);
  for (int k = -200; k <= 200; k++)
    for (double sg : {1.0, -1.0}) {
      const double a = sg * (edge + k * 1e-12), yaw = 0.3 * k;
      s.rpy(0, a, 0);
      s.rpy(0.1, a, yaw);
    }

  // matrices entered directly: m[2][0] at, beyond and just inside +-1, and random entries for every getRotation branch
  for (int n = 0; n < 4000; n++) {
    double m[3][3], o[3] = {u(rng), u(rng), u(rng)};
    for (auto &r : m)
      for (double &x : r) x = u(rng);
    const double m20[] = {1.0, -1.0, std::nextafter(1.0, 0.0), std::nextafter(-1.0, 0.0), std::nextafter(1.0, 2.0),
                          std::nextafter(-1.0, -2.0)};
    if (n < 600) m[2][0] = m20[n % 6];
    s.entries(m, o);
  }

  // chains of products and inverses, and Transform::operator()(v)
  for (int chain = 0; chain < 300; chain++) {
    double q[4] = {u(rng), u(rng), u(rng), u(rng)}, o[3] = {big(rng) * 1e-4, big(rng) * 1e-4, big(rng) * 1e-4};
    double q2[ROS_MATH_CHAIN_STEPS][4], o2[ROS_MATH_CHAIN_STEPS][3], v[ROS_MATH_CHAIN_STEPS][3];
    for (int step = 0; step < ROS_MATH_CHAIN_STEPS; step++) {
      for (double &x : q2[step]) x = u(rng);
      for (double &x : o2[step]) x = u(rng) * 10;
      for (double &x : v[step]) x = u(rng) * 5;
    }
    s.chain(q, o, q2, o2, v);
  }

  // stamps: negative and overflowing nanoseconds, seconds across the int32 wrap.  A nanosecond field is below 2^31:
  // roscpp subtracts the fields as int32, which overflows beyond that.
  const uint32_t secs[] = {0, 1, 2, 1000, 0x7ffffffeu, 0x7fffffffu, 0x80000000u, 0x80000001u, 0xfffffffeu, 0xffffffffu};
  const uint32_t nsecs[] = {0, 1, 999999999u, 1000000000u, 1000000001u, 1999999999u, 2000000000u, 0x7fffffffu, 500000000u};
  for (uint32_t s1 : secs)
    for (uint32_t s0 : secs)
      for (uint32_t n1 : nsecs)
        for (uint32_t n0 : nsecs) s.stamps(s1, n1, s0, n0);
  for (int n = 0; n < 20000; n++) {
    const uint32_t s1 = any32(rng), n1 = any32(rng) >> 1, s0 = any32(rng), n0 = any32(rng) >> 1;
    s.stamps(s1, n1, s0, n0);
  }

  // Duration::fromSec: x.9999999995 (rolls a second over), negative values, random values, and the comparison
  const double secs_d[] = {0.0, -0.0, 0.9999999995, 1.9999999995, 41.9999999995, -0.0000000005, -1e-10, -0.5,
                           -1.0, -2.5, -3.9999999995, -1.0000000005, 0.0000000005, 1e-10, 2147483647.0, -2147483648.0,
                           0.99999999949999, 0.9999999994999999, 1.25, 3.0000000004999};
  for (double d : secs_d) s.from_sec(d);
  for (int n = 0; n < 20000; n++) {
    const double d = n % 2 ? big(rng) : std::floor(big(rng)) + (n % 4 == 1 ? 0.9999999995 : -0.0000000005);
    const double d2 = n % 3 ? big(rng) : d;
    s.from_sec_pair(d, d2);
  }
}
