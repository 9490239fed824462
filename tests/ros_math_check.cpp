// TEST HELPER (host only): the three definitions of tf / tf2 LinearMath and roscpp Time / Duration — the library's
// csrc/ros_math.cuh, the C restatements' oracle/linear_math.h and the node stand-ins' classes (oracle/shim/tf2,
// oracle/shim/tf, oracle/shim_lesson6/tf/tf_core.h, oracle/shim/ros/ros.h) — on the seeded sweep of inputs of
// ros_math_sweep.h, compared bit for bit (a NaN matches any NaN).  Prints one JSON line: checks, mismatches, the first mismatch, and how often each
// branch of the restated code was taken.  Build with -ffp-contract=off, as the library's host code and the stand-ins.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/ros_math.cuh"
#include "../oracle/linear_math.h"
#include "ros_math_sweep.h"
#include "ros/ros.h"
#include "tf/LinearMath/Matrix3x3.h"
#include "tf/tf_core.h"
#include "tf2/utils.h"

namespace {

long checks = 0, mismatches = 0;
std::string first;
std::map<std::string, long> branches;

bool same(double a, double b) { return (std::isnan(a) && std::isnan(b)) || std::memcmp(&a, &b, sizeof a) == 0; }

void expect(const char *what, int idx, double lib, double c, double shim) {
  checks++;
  if (same(lib, c) && same(lib, shim)) return;
  if (!mismatches++) {
    char buf[256];
    std::snprintf(buf, sizeof buf, "%s[%d]: library %.17g, C %.17g, stand-in %.17g", what, idx, lib, c, shim);
    first = buf;
  }
}
void expect2(const char *what, int idx, double lib, double shim) { expect(what, idx, lib, lib, shim); }

struct Three {
  b2s::TfTransform lib;
  orc_tf c;
  tf2::Transform shim;
};

Three from_entries(const double m[3][3], const double o[3]) {
  Three t;
  std::memcpy(t.lib.m, m, sizeof t.lib.m);
  std::memcpy(t.lib.o, o, sizeof t.lib.o);
  std::memcpy(&t.c, &t.lib, sizeof t.c);
  t.shim = tf2::Transform(tf2::Matrix3x3(m[0][0], m[0][1], m[0][2], m[1][0], m[1][1], m[1][2], m[2][0], m[2][1], m[2][2]),
                          tf2::Vector3(o[0], o[1], o[2]));
  return t;
}

Three from_quaternion(const double q[4], const double o[3]) {
  Three t;
  b2s::tf_set_rotation(t.lib, q);
  std::memcpy(t.lib.o, o, sizeof t.lib.o);
  tf_set_rotation(&t.c, q);
  std::memcpy(t.c.o, o, sizeof t.c.o);
  t.shim.setRotation(tf2::Quaternion(q[0], q[1], q[2], q[3]));
  t.shim.setOrigin(tf2::Vector3(o[0], o[1], o[2]));
  return t;
}

void compare(const char *what, const Three &t) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) expect(what, 3 * i + j, t.lib.m[i][j], t.c.m[i][j], t.shim.getBasis()[i][j]);
    expect(what, 9 + i, t.lib.o[i], t.c.o[i], t.shim.getOrigin()[i]);
  }
}

// getRotation, getRPY and tf2's getYaw of the rotation, counting the branches the library takes
void check_rotation(const Three &t) {
  const double(*m)[3] = t.lib.m;
  const double trace = m[0][0] + m[1][1] + m[2][2];
  branches[trace > 0.0 ? "get_rotation_trace" : m[0][0] < m[1][1] ? (m[1][1] < m[2][2] ? "get_rotation_i2" : "get_rotation_i1")
                                                                   : (m[0][0] < m[2][2] ? "get_rotation_i2" : "get_rotation_i0")]++;
  double ql[4], qc[4];
  b2s::tf_get_rotation(t.lib, ql);
  tf_get_rotation(&t.c, qc);
  const tf2::Quaternion qs = t.shim.getRotation();
  for (int k = 0; k < 4; k++) expect("getRotation", k, ql[k], qc[k], qs.q[k]);

  branches[std::fabs(m[2][0]) >= 1 ? (m[2][0] > 0 ? "get_rpy_singular_up" : "get_rpy_singular_down") : "get_rpy"]++;
  double rl[3], rc[3], rs[3];
  b2s::tf_get_rpy(t.lib, rl[0], rl[1], rl[2]);
  tf_get_rpy(&t.c, &rc[0], &rc[1], &rc[2]);
  t.shim.getBasis().getRPY(rs[0], rs[1], rs[2]);
  for (int k = 0; k < 3; k++) expect("getRPY", k, rl[k], rc[k], rs[k]);

  const double sqx = ql[0] * ql[0], sqy = ql[1] * ql[1], sqz = ql[2] * ql[2], sqw = ql[3] * ql[3];
  const double sarg = -2 * (ql[0] * ql[2] - ql[3] * ql[1]) / (sqx + sqy + sqz + sqw);
  branches[sarg <= -0.99999 ? "tf2_yaw_sarg_low" : sarg >= 0.99999 ? "tf2_yaw_sarg_high" : "tf2_yaw"]++;
  expect("tf2::getYaw", 0, b2s::tf2_get_yaw(ql), tf2_get_yaw(qc), tf2::getYaw(qs));
}

// everything computed from a quaternion: setRotation (and the Matrix3x3(q) constructor), tf::getYaw, then the rotation
void check_quaternion(const double q[4]) {
  const double o[3] = {0, 0, 0};
  const Three t = from_quaternion(q, o);
  compare("setRotation", t);
  const tf2::Matrix3x3 mq(tf2::Quaternion(q[0], q[1], q[2], q[3]));
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) expect2("Matrix3x3(q)", 3 * i + j, t.lib.m[i][j], mq[i][j]);
  double roll, pitch, yaw;
  tf_get_rpy(&t.c, &roll, &pitch, &yaw);
  expect("tf::getYaw", 0, b2s::tf_get_yaw(q), yaw, tf::getYaw(tf::Quaternion(q[0], q[1], q[2], q[3])));
  check_rotation(t);
}

void check_rpy(double r, double p, double y) {
  double ql[4], qc[4];
  b2s::quat_set_rpy(r, p, y, ql);
  quat_set_rpy(r, p, y, qc);
  tf2::Quaternion qs;
  qs.setRPY(r, p, y);
  const tf::Quaternion qt = tf::createQuaternionFromRPY(r, p, y);
  for (int k = 0; k < 4; k++) {
    expect("setRPY", k, ql[k], qc[k], qs.q[k]);
    expect2("createQuaternionFromRPY", k, ql[k], qt.q[k]);
  }
  check_quaternion(ql);
}

void check_stamps(uint32_t s1, uint32_t n1, uint32_t s0, uint32_t n0) {
  const b2s::RosDuration dl = b2s::ros_time_diff(s1, n1, s0, n0);
  const orc_duration dc = ros_time_diff(s1, n1, s0, n0);
  const ros::Duration ds = ros::Time(s1, n1) - ros::Time(s0, n0);
  const ros::Duration dm = ros::Time(s1, n1).operator ros::Time::Stamp() - ros::Time(s0, n0);  // Stamp - Time
  branches[(int64_t)(int32_t)n1 - (int32_t)n0 < 0 ? "time_diff_nsec_negative" : "time_diff_nsec_positive"]++;
  if ((int64_t)(int32_t)s1 - (int32_t)s0 != (int32_t)(s1 - s0)) branches["time_diff_sec_wraps"]++;
  expect("Time-Time sec", 0, dl.sec, dc.sec, ds.sec);
  expect("Time-Time nsec", 0, dl.nsec, dc.nsec, ds.nsec);
  expect2("Stamp-Time", 0, dl.sec, dm.sec);
  expect2("Stamp-Time", 1, dl.nsec, dm.nsec);
  expect("Duration::toSec", 0, b2s::ros_duration_to_sec(dl), ros_duration_to_sec(dc), ds.toSec());
  ros::Time::Stamp st = ros::Time(s1, n1);
  expect("Time::toSec", 0, b2s::ros_time_to_sec(s1, n1), ros_time_to_sec(s1, n1), st.toSec());
}

void check_from_sec(double d) {
  const b2s::RosDuration dl = b2s::ros_duration_from_sec(d);
  const ros::Duration ds(d);
  if (std::round((d - std::floor(d)) * 1e9) >= 1e9) branches["from_sec_rollover"]++;
  if (d < 0) branches["from_sec_negative"]++;
  expect2("fromSec sec", 0, dl.sec, ds.sec);
  expect2("fromSec nsec", 0, dl.nsec, ds.nsec);
}

void check_compare(const b2s::RosDuration &a, const b2s::RosDuration &b) {
  expect2("Duration>", 0, b2s::ros_duration_gt(a, b), ros::Duration(a.sec, a.nsec) > ros::Duration(b.sec, b.nsec));
}

// the sweep's sink: every input through all three definitions
struct Checks {
  void quaternion(const double q[4]) { check_quaternion(q); }
  void rpy(double r, double p, double y) { check_rpy(r, p, y); }
  void entries(const double m[3][3], const double o[3]) { check_rotation(from_entries(m, o)); }
  void chain(const double q[4], const double o[3], const double q2[][4], const double o2[][3], const double v[][3]) {
    Three acc = from_quaternion(q, o);
    for (int step = 0; step < ROS_MATH_CHAIN_STEPS; step++) {
      const Three b = from_quaternion(q2[step], o2[step]);
      Three next;
      if (step % 3 == 0) {  // acc * b^-1
        const b2s::TfTransform il = b2s::tf_inverse(b.lib);
        const orc_tf ic = tf_inverse(&b.c);
        next.lib = b2s::tf_mul(acc.lib, il);
        next.c = tf_mul(&acc.c, &ic);
        next.shim = acc.shim * b.shim.inverse();
      } else if (step % 3 == 1) {  // b * acc
        next.lib = b2s::tf_mul(b.lib, acc.lib);
        next.c = tf_mul(&b.c, &acc.c);
        next.shim = b.shim * acc.shim;
      } else {  // (acc * b)^-1
        const b2s::TfTransform pl = b2s::tf_mul(acc.lib, b.lib);
        const orc_tf pc = tf_mul(&acc.c, &b.c);
        next.lib = b2s::tf_inverse(pl);
        next.c = tf_inverse(&pc);
        next.shim = (acc.shim * b.shim).inverse();
      }
      acc = next;
      compare("product / inverse", acc);
      double vl[3];
      b2s::tf_apply(acc.lib, v[step], vl);
      const tf2::Vector3 vs = acc.shim(tf2::Vector3(v[step][0], v[step][1], v[step][2]));
      for (int i = 0; i < 3; i++) expect2("Transform(v)", i, vl[i], vs[i]);
      check_rotation(acc);
    }
    Three id;
    b2s::tf_identity(id.lib);
    tf_identity(&id.c);
    id.shim = tf2::Transform();
    compare("identity", id);
  }
  void stamps(uint32_t s1, uint32_t n1, uint32_t s0, uint32_t n0) { check_stamps(s1, n1, s0, n0); }
  void from_sec(double d) { check_from_sec(d); }
  void from_sec_pair(double d, double d2) {
    check_from_sec(d);
    const b2s::RosDuration a = b2s::ros_duration_from_sec(d), b = b2s::ros_duration_from_sec(d2);
    check_compare(a, b);
    check_compare(b, a);
  }
};

}  // namespace

int main() {
  Checks checks_sink;
  ros_math_sweep(checks_sink);

  std::printf("{\"checks\": %ld, \"mismatches\": %ld, \"first\": \"%s\", \"branches\": {", checks, mismatches, first.c_str());
  const char *sep = "";
  for (const auto &b : branches) {
    std::printf("%s\"%s\": %ld", sep, b.first.c_str(), b.second);
    sep = ", ";
  }
  std::printf("}}\n");
  return 0;
}
