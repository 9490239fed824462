/*
 * ref_lesson6.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson6 node, reference/lesson6/src/karto_slam.cc, #included where it lies,
 * linked with the unmodified open_karto Karto.cpp / Mapper.cpp (oracle/recipes.py builds _ref/liblesson6_ref.so).
 * ROS, tf and Boost threads are absent; the stand-ins under oracle/shim_lesson6/ (first on the include path: Boost,
 * message_filters, tf's listener and Stamped, the message types only this node uses) and oracle/shim/ provide the node handle and its parameters, ros::Time / Duration, the publishers (a hook per message
 * type), tf's LinearMath, a listener answering from the mount and the odometry the driver sets, and Boost's bind,
 * mutex and thread.  The node's main() is renamed so the library has none; every line of the node that runs here is the
 * reference's.  LaserScans go in through the public laserCallback; the published maps and the state they came from come
 * back out.
 *
 * karto_slam.h includes the four back-end headers by quote, next to it, and they need Eigen, sba, g2o, Ceres and GTSAM.
 * Their include guards are defined here and SpaSolver / G2oSolver / CeresSolver / GTSAMSolver declared instead: each is
 * a karto::ScanSolver forwarding to the C callbacks of a b2s_scan_solver (as ref_driver.cpp's CallbackSolver does), so a
 * test plugs the same back end into the node and into the library.  SpaSolver::getGraph returns no vertices, so the
 * node's graph markers stay empty.
 *
 * The node's header is included with `private` spelled `public`, after every other header it pulls in, so that only
 * the node's class is affected.
 */
#include <cstring>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <queue>
#include <set>
#include <sstream>
#include <string>
#include <vector>

#include <ros/ros.h>
#include <ros/console.h>
#include <boost/thread.hpp>
#include <message_filters/subscriber.h>
#include <tf/transform_broadcaster.h>
#include <tf/transform_listener.h>
#include <tf/message_filter.h>
#include <visualization_msgs/MarkerArray.h>
#include <sensor_msgs/LaserScan.h>
#include <nav_msgs/MapMetaData.h>
#include <nav_msgs/GetMap.h>
#include <open_karto/Mapper.h>

#include "../include/b200slam.h"

namespace {

b2s_scan_solver g_solver;  // the back end the node's CreateSolver gets

struct CallbackSolver : karto::ScanSolver {
  b2s_scan_solver cb = g_solver;
  IdPoseVector corrections;
  int n_nodes = 0;
  void Compute() override {
    corrections.clear();
    std::vector<int32_t> ids(n_nodes);
    std::vector<double> poses(3 * static_cast<size_t>(n_nodes));
    int n = cb.compute(cb.user, n_nodes, ids.data(), poses.data());
    for (int i = 0; i < n; i++)
      corrections.push_back(std::make_pair(ids[i], karto::Pose2(poses[3 * i], poses[3 * i + 1], poses[3 * i + 2])));
  }
  const IdPoseVector &GetCorrections() const override { return corrections; }
  void AddNode(karto::Vertex<karto::LocalizedRangeScan> *v) override {
    karto::Pose2 p = v->GetObject()->GetCorrectedPose();
    double c[3] = {p.GetX(), p.GetY(), p.GetHeading()};
    n_nodes++;
    cb.add_node(cb.user, v->GetObject()->GetUniqueId(), c);
  }
  void AddConstraint(karto::Edge<karto::LocalizedRangeScan> *e) override {
    karto::LinkInfo *li = (karto::LinkInfo *)(e->GetLabel());
    karto::Pose2 d = li->GetPoseDifference();
    double diff[3] = {d.GetX(), d.GetY(), d.GetHeading()}, cov[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cov[3 * i + j] = li->GetCovariance()(i, j);
    cb.add_constraint(cb.user, e->GetSource()->GetObject()->GetUniqueId(), e->GetTarget()->GetObject()->GetUniqueId(), diff,
                      cov);
  }
  void Clear() override {
    corrections.clear();
    if (cb.clear) cb.clear(cb.user);
  }
};

}  // namespace

#define LESSON6_SPA_SOLVER_H
#define KARTO_G2OSOLVER_H
#define LESSON6_CERES_SOLVER_CERES_SOLVER_H
#define KARTO_GTSAM_SOLVER_H_
struct SpaSolver : CallbackSolver {
  void getGraph(std::vector<float> &) {}
};
struct G2oSolver : CallbackSolver {};
struct CeresSolver : CallbackSolver {};
struct GTSAMSolver : CallbackSolver {};

#define private public
#include <lesson6/karto_slam.h>
#undef private

#define main lesson6_karto_slam_main
#include "lesson6/src/karto_slam.cc"
#undef main

namespace {

int g_node_counter = 0;

struct NullBuf : std::streambuf {
  int overflow(int c) override { return c; }
};
// open_karto prints "Registering sensor" etc. on std::cout; keep test logs clean
struct CoutSilencer {
  NullBuf nb;
  std::streambuf *old;
  CoutSilencer() : old(std::cout.rdbuf(&nb)) {}
  ~CoutSilencer() { std::cout.rdbuf(old); }
};

struct Run {
  SlamKarto *node = nullptr;
  std::string frame;
  tf::Transform mount;
};

tf::Transform from_row(const double *r) {
  return tf::Transform(tf::Quaternion(r[3], r[4], r[5], r[6]), tf::Vector3(r[0], r[1], r[2]));
}

int processed_count(SlamKarto *n) {
  return static_cast<int>(n->mapper_->GetAllProcessedScans().size());
}

}  // namespace

extern "C" {

typedef void (*ref_map_fn)(void *user, int32_t width, int32_t height, float resolution, double origin_x, double origin_y,
                           const int8_t *payload);

/* clear the parameter server; ref_karto_param / _param_str set one value; ref_karto_set_solver names the back end the
 * next node's CreateSolver gets (NULL: none, then use_back_end must be false) */
void ref_karto_clear_params() {
  ros::shim::params().clear();
  ros::shim::string_params().clear();
}
void ref_karto_param(const char *name, double value) { ros::shim::params()[name] = value; }
void ref_karto_param_str(const char *name, const char *value) { ros::shim::string_params()[name] = value; }
void ref_karto_set_solver(const b2s_scan_solver *s) {
  if (s) g_solver = *s;
  else std::memset(&g_solver, 0, sizeof g_solver);
}

/* a fresh node with the parameters set so far; mount = base_link <- laser as translation xyz + quaternion xyzw.  Each
 * node gets its own laser frame id (karto's SensorManager is process-wide).  Nodes are never destroyed: ~SlamKarto
 * deletes solver_, which the node leaves uninitialised without a back end. */
void *ref_karto_new(const double mount[7]) {
  CoutSilencer quiet;
  Run *r = new Run();
  std::stringstream nm;
  nm << "laser_" << (g_node_counter++);
  r->frame = nm.str();
  r->mount = from_row(mount);
  r->node = new SlamKarto();
  return r;
}

/* laserCallback on one LaserScan; fields[5] = angle_min, angle_max, angle_increment, range_min, range_max; odom = the
 * odom <- base_link transform at its stamp (a NaN: the lookup throws).  Outputs as b2s_karto_node_process's for one
 * scan; every map the node publishes goes to on_map.  Returns 0, or -1 when the callback threw. */
int ref_karto_scan(void *h, uint32_t sec, uint32_t nsec, const float fields[5], int n, const float *ranges,
                   const double odom[7], int32_t *out_state, double out_pose[3], double out_m2o[7], int32_t *out_published,
                   ref_map_fn on_map, void *user) {
  CoutSilencer quiet;
  Run *r = static_cast<Run *>(h);
  SlamKarto *node = r->node;
  auto m = std::make_shared<sensor_msgs::LaserScan>();
  m->header.stamp.sec = sec;
  m->header.stamp.nsec = nsec;
  m->header.frame_id = r->frame;
  m->angle_min = fields[0];
  m->angle_max = fields[1];
  m->angle_increment = fields[2];
  m->range_min = fields[3];
  m->range_max = fields[4];
  m->ranges.assign(ranges, ranges + n);
  sensor_msgs::LaserScan::ConstPtr c = m;
  tf::shim::Frames &f = tf::shim::frames();
  f.base_laser = r->mount;
  f.odom_ok = true;
  for (int k = 0; k < 7; k++) f.odom_ok = f.odom_ok && !std::isnan(odom[k]);
  if (f.odom_ok) f.odom_base = from_row(odom);
  const int failures_before = f.odom_failures, processed_before = processed_count(node);
  int published = 0;
  ros::shim::on_publish<nav_msgs::OccupancyGrid>() = [&](const nav_msgs::OccupancyGrid &g) {
    published++;
    if (on_map)
      on_map(user, (int32_t)g.info.width, (int32_t)g.info.height, g.info.resolution, g.info.origin.position.x,
             g.info.origin.position.y, g.data.data());
  };
  try {
    node->laserCallback(c);
  } catch (const std::exception &) {
    ros::shim::on_publish<nav_msgs::OccupancyGrid>() = nullptr;
    return -1;
  }
  ros::shim::on_publish<nav_msgs::OccupancyGrid>() = nullptr;
  const bool throttled = (node->laser_count_ % node->throttle_scans_) != 0;
  const int processed_after = processed_count(node);
  *out_state = throttled ? B2S_KARTO_THROTTLED
                         : (f.odom_failures != failures_before ? B2S_KARTO_NO_ODOM
                                                              : (processed_after > processed_before ? B2S_KARTO_PROCESSED
                                                                                                    : B2S_KARTO_NOT_MOVED));
  out_pose[0] = out_pose[1] = out_pose[2] = 0;
  if (*out_state == B2S_KARTO_PROCESSED) {
    karto::Pose2 p = node->mapper_->GetAllProcessedScans().back()->GetCorrectedPose();
    out_pose[0] = p.GetX();
    out_pose[1] = p.GetY();
    out_pose[2] = p.GetHeading();
  }
  const tf::Vector3 o = node->map_to_odom_.getOrigin();
  const tf::Quaternion q = node->map_to_odom_.getRotation();
  out_m2o[0] = o.x(); out_m2o[1] = o.y(); out_m2o[2] = o.z();
  out_m2o[3] = q.x(); out_m2o[4] = q.y(); out_m2o[5] = q.z(); out_m2o[6] = q.w();
  *out_published = published;
  return 0;
}

/* the node's graph: processed scans' corrected poses in unique-id order [count][3]; edges as b2s_mapper_get_edges */
int ref_karto_scan_count(void *h) { return processed_count(static_cast<Run *>(h)->node); }
void ref_karto_poses(void *h, double *out) {
  karto::Mapper *mp = static_cast<Run *>(h)->node->mapper_;
  const int n = processed_count(static_cast<Run *>(h)->node);
  for (int i = 0; i < n; i++) {
    karto::Pose2 c = mp->GetMapperSensorManager()->GetScan(i)->GetCorrectedPose();
    out[3 * i] = c.GetX(); out[3 * i + 1] = c.GetY(); out[3 * i + 2] = c.GetHeading();
  }
}
int ref_karto_edge_count(void *h) {
  karto::Mapper *mp = static_cast<Run *>(h)->node->mapper_;
  return mp->GetGraph() ? static_cast<int>(mp->GetGraph()->GetEdges().size()) : 0;
}
void ref_karto_edges(void *h, int32_t *ids, double *diff, double *cov) {
  karto::Mapper *mp = static_cast<Run *>(h)->node->mapper_;
  const std::vector<karto::Edge<karto::LocalizedRangeScan> *> &e = mp->GetGraph()->GetEdges();
  for (size_t i = 0; i < e.size(); i++) {
    karto::LinkInfo *li = (karto::LinkInfo *)(e[i]->GetLabel());
    ids[2 * i] = e[i]->GetSource()->GetObject()->GetUniqueId();
    ids[2 * i + 1] = e[i]->GetTarget()->GetObject()->GetUniqueId();
    karto::Pose2 d = li->GetPoseDifference();
    diff[3 * i] = d.GetX(); diff[3 * i + 1] = d.GetY(); diff[3 * i + 2] = d.GetHeading();
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) cov[9 * i + 3 * r + c] = li->GetCovariance()(r, c);
  }
}

}  // extern "C"
