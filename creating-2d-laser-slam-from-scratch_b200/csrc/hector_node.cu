// lesson4's HectorMappingRos node (lesson4/src/hector_mapping/hector_slam.cc) over a whole recording of one laser: host
// C++ around the device HectorSlamProcessor (hector_slam.cu), whose k_hs_stream_node converts and matches the scans.
//   HectorMappingRos::InitParams / constructor       hector_slam.cc:26-105, 119-162
//   HectorMappingRos::setMapInfo                     :165-180
//   HectorMappingRos::scanCallback                   :186-251  (projectLaser, rosPointCloudToDataContainer, update)
//   PoseInfoContainer::update                        util/PoseInfoContainer.h:53-92
//   HectorMappingRos::publishMapLoop / publishMap    :254-317  (level 0 only, the update-index gate)
// tf's LinearMath and roscpp's Time / Duration are ros_math.cuh's (include/b200slam.h, DESIGN.md §7).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <memory>
#include <new>
#include <vector>

#include "common.cuh"
#include "hector_scan.cuh"
#include "ros_math.cuh"

namespace b2s {
// hector_slam.cu
void hs_node_map_info(const b2s_hector_slam *p, float &origin_x, float &origin_y, float &cell_length, int &w, int &h);
float hs_scale_to_map(const b2s_hector_slam *p);
b2s_status hs_node_run(b2s_hector_slam *p, HsNodeIo &io, const b2s_laser_scan_msg &geometry, const double *units,
                       double range_cutoff, const HectorNodeFilter &filter, int n_scans, const float *ranges,
                       const std::vector<int> &cuts, float *out_rows,
                       const std::function<b2s_status(size_t, const int8_t *)> &on_map);
}  // namespace b2s

using namespace b2s;

namespace {
constexpr int NODE_MAX_RANGES = 4096;      // the processor's per-scan capacity
constexpr int NODE_MAX_SCANS = (1 << 20) - 1;  // stamp epochs of one call (hector_slam.cu)
constexpr int64_t NS = 1000000000LL;

int64_t stamp_ns(const uint32_t *s) { return (int64_t)s[0] * NS + (int64_t)s[1]; }
}  // namespace

struct b2s_hector_node {
  b2s_hector_node_params prm{};
  b2s_laser_scan_msg geom{};
  int device = 0;
  b2s_hector_slam *proc = nullptr;
  HectorNodeFilter filter{};
  double cutoff = 30.0;  // projector_.projectLaser(scan, laser_point_cloud_, 30.0)
  std::vector<double> units;
  int64_t period_ns = 0;            // Duration::fromSec(map_pub_period)
  bool started = false;             // tick 0 set (a scan was handed in)
  int64_t next_tick_ns = 0;
  int64_t scans = 0;                // scans handed in so far
  int64_t updates = 0;              // map updates so far: level 0's getUpdateIndex() = updates - 1
  int64_t last_get_map_update_index = -100;  // lastGetMapUpdateIndex
  b2s_hector_node_map_info info{};
  HsNodeIo io;
  std::vector<float> rows;
  std::vector<int8_t> payload;      // b2s_hector_node_publish_map's
  bool failed = false;              // a call failed partway: maps were handed out, the schedule was not committed
};

namespace {

// publishMap's gate: rebuild when the grid's update index moved since the last publish
int32_t map_gate(b2s_hector_node *n, int64_t updates) {
  const int64_t index = updates - 1;
  const bool rebuilt = index != n->last_get_map_update_index;
  n->last_get_map_update_index = index;
  return rebuilt ? 1 : 0;
}

}  // namespace

extern "C" {

b2s_status b2s_hector_node_create(const b2s_hector_node_params *params, const b2s_laser_scan_msg *geometry,
                                  const double laser_mount[7], int device, b2s_hector_node **out) {
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: null argument");
  *out = nullptr;
  if (!params || !geometry || !laser_mount) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: null argument");
  const float res = static_cast<float>(params->map_resolution);
  if (!(res > 0.0f) || !std::isfinite(res)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: map_resolution must be positive");
  if (params->map_size <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: map_size must be positive");
  const double period = params->map_pub_period;
  if (!(period > 0.0) || !std::isfinite(period) || std::floor(period) > 2147483647.0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: map_pub_period must be positive, finite and inside ros::Duration's range");
  const RosDuration d = ros_duration_from_sec(period);
  const int64_t period_ns = (int64_t)d.sec * NS + (int64_t)d.nsec;
  if (period_ns <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: map_pub_period rounds to a zero ros::Duration");
  if (geometry->angle_increment == 0.0f || geometry->n_ranges < 0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: zero angle_increment or negative n_ranges");
  if (geometry->n_ranges > NODE_MAX_RANGES) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_hector_node_create: at most 4096 ranges per scan");
  double qn = 0.0;
  for (int k = 0; k < 7; k++)
    if (!std::isfinite(laser_mount[k])) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: non-finite laser mount");
  for (int k = 3; k < 7; k++) qn += laser_mount[k] * laser_mount[k];
  if (!(qn > 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_create: zero mount quaternion");

  // the constructor: HectorSlamProcessor(static_cast<float>(resolution), size, size, Vector2f(start), levels) + setters
  b2s_hector_slam *proc = nullptr;
  if (b2s_status st = b2s_hector_slam_create_batch(1, std::max(geometry->n_ranges, 1), res, params->map_size,
                                                   params->map_size, static_cast<float>(params->map_start_x),
                                                   static_cast<float>(params->map_start_y),
                                                   params->map_multi_res_levels, device, nullptr, &proc))
    return st;
  b2s_status st = b2s_hector_slam_set_update_factors(proc, static_cast<float>(params->update_factor_free),
                                                      static_cast<float>(params->update_factor_occupied));
  if (!st)
    st = b2s_hector_slam_set_map_update_min_diff(proc, static_cast<float>(params->map_update_distance_thresh),
                                                 static_cast<float>(params->map_update_angle_thresh));
  if (st) {
    b2s_hector_slam_destroy(proc);
    return st;
  }
  b2s_hector_node *n = new (std::nothrow) b2s_hector_node();
  if (!n) {
    b2s_hector_slam_destroy(proc);
    B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  }
  std::unique_ptr<b2s_hector_node, decltype(&b2s_hector_node_destroy)> guard(n, b2s_hector_node_destroy);
  n->prm = *params;
  n->geom = *geometry;
  n->geom.ranges = nullptr;
  n->device = device;
  n->proc = proc;
  n->period_ns = period_ns;
  // rosPointCloudToDataContainer's settings: the thresholds as InitParams stores them, the mount's tf::Transform
  HectorNodeFilter &f = n->filter;
  f.sqr_min = static_cast<float>(params->laser_min_dist * params->laser_min_dist);
  f.sqr_max = static_cast<float>(params->laser_max_dist * params->laser_max_dist);
  f.use_max_scan_range = params->use_max_scan_range;
  tf_set_rotation(f.mount, laser_mount + 3);
  f.mount.o[0] = laser_mount[0]; f.mount.o[1] = laser_mount[1]; f.mount.o[2] = laser_mount[2];
  f.z_min = params->laser_z_min_value;
  f.z_max = params->laser_z_max_value;
  f.scale_to_map = hs_scale_to_map(proc);
  n->units.resize(2 * (size_t)std::max(geometry->n_ranges, 1));
  hector_unit_vectors(geometry->angle_min, geometry->angle_increment, geometry->n_ranges, n->units.data());
  float ox, oy, cl;
  int w, h;
  hs_node_map_info(proc, ox, oy, cl, w, h);
  n->info.origin_x = ox; n->info.origin_y = oy;
  n->info.resolution = cl;
  n->info.width = w; n->info.height = h;
  B2S_CUDA_CHECK(cudaSetDevice(device));
  B2S_CUDA_CHECK(n->io.copy.init(nullptr));
  for (int k = 0; k < 2; k++) {
    B2S_CUDA_CHECK(n->io.converted[k].create(cudaEventDisableTiming));
    B2S_CUDA_CHECK(n->io.copied[k].create(cudaEventDisableTiming));
  }
  *out = guard.release();
  return B2S_OK;
}

void b2s_hector_node_destroy(b2s_hector_node *n) {
  if (!n) return;
  if (n->proc) {
    cudaSetDevice(n->device);
    if (n->io.copy.s) cudaStreamSynchronize(n->io.copy);
    b2s_hector_slam_destroy(n->proc);
  }
  delete n;
}

b2s_hector_slam *b2s_hector_node_processor(b2s_hector_node *n) { return n ? n->proc : nullptr; }

b2s_status b2s_hector_node_process(b2s_hector_node *n, int n_scans, const float *ranges, const uint32_t *stamps,
                                   float *out_pose, double *out_pose_msg, double *out_cov, int32_t *out_map_updated,
                                   int32_t *out_n_points, b2s_hector_node_map_fn on_map, void *user) {
  B2S_NVTX("HectorMappingRos::scanCallback");
  if (!n || n_scans < 0 || (n_scans > 0 && (!stamps || (!ranges && n->geom.n_ranges > 0))))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_process: null argument or negative count");
  if (n->failed) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_node_process: an earlier call failed partway; destroy the handle");
  if (n_scans >= NODE_MAX_SCANS) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_hector_node_process: too many scans in one call (split it)");
  if (n_scans == 0) return B2S_OK;
  // the schedule: the scans a publish precedes, and their ticks
  std::vector<int> cuts;
  std::vector<int64_t> ticks;
  bool started = n->started;
  int64_t next = n->next_tick_ns;
  for (int i = 0; i < n_scans; i++) {
    const int64_t s = stamp_ns(stamps + 2 * (size_t)i);
    if (!started) {
      started = true;
      next = s;  // tick 0
    }
    if (s >= next) {
      cuts.push_back(i);
      ticks.push_back(next);
      next += ((s - next) / n->period_ns + 1) * n->period_ns;  // the first tick strictly after s
    }
  }
  n->rows.resize(16 * (size_t)n_scans);
  int64_t counted = 0, updates = n->updates;  // flags of the call's scans [0, counted) are in `updates`
  auto publish = [&](size_t k, const int8_t *payload) -> b2s_status {
    const float *rows = n->io.h_rows;
    for (; counted < cuts[k]; counted++) updates += rows[16 * (size_t)counted + 12] != 0.0f ? 1 : 0;
    const int32_t rebuilt = map_gate(n, updates);
    const uint32_t stamp[2] = {(uint32_t)(ticks[k] / NS), (uint32_t)(ticks[k] % NS)};
    if (on_map) on_map(user, (int32_t)(n->scans + cuts[k]), stamp, &n->info, payload, rebuilt);
    return B2S_OK;
  };
  b2s_status st = hs_node_run(n->proc, n->io, n->geom, n->units.data(), n->cutoff, n->filter, n_scans, ranges, cuts,
                              n->rows.data(), publish);
  if (st) {
    // the processor, the maps handed out and the publish gate have moved, the schedule and the counters have not
    n->failed = true;
    return st;
  }
  n->started = started;
  n->next_tick_ns = next;
  for (int i = 0; i < n_scans; i++) {
    const float *r = n->rows.data() + 16 * (size_t)i;
    const bool upd = r[12] != 0.0f;
    n->updates += upd ? 1 : 0;
    if (out_pose) std::memcpy(out_pose + 3 * (size_t)i, r, 3 * sizeof(float));
    if (out_pose_msg) {
      // PoseInfoContainer::update: position x / y, orientation w = cos(yaw * 0.5f), z = sin(yaw * 0.5f) (double calls)
      double *m = out_pose_msg + 7 * (size_t)i;
      const float half = r[2] * 0.5f;
      m[0] = (double)r[0]; m[1] = (double)r[1]; m[2] = 0.0;
      m[3] = 0.0; m[4] = 0.0; m[5] = sin((double)half); m[6] = cos((double)half);
    }
    if (out_cov) {
      const float *h = r + 3;  // row-major 3x3
      double *c = out_cov + 36 * (size_t)i;
      for (int q = 0; q < 36; q++) c[q] = 0.0;
      c[0] = (double)h[0]; c[7] = (double)h[4]; c[35] = (double)h[8];
      c[1] = c[6] = (double)h[1];
      c[5] = c[30] = (double)h[2];
      c[11] = c[31] = (double)h[5];
    }
    if (out_map_updated) out_map_updated[i] = upd ? 1 : 0;
    if (out_n_points) std::memcpy(out_n_points + i, r + 15, sizeof(int32_t));
  }
  n->scans += n_scans;
  return B2S_OK;
}

b2s_status b2s_hector_node_publish_map(b2s_hector_node *n, const uint32_t stamp[2], b2s_hector_node_map_fn on_map,
                                       void *user) {
  if (!n || !stamp) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_publish_map: null argument");
  if (n->failed) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_node_publish_map: an earlier call failed partway; destroy the handle");
  n->payload.resize((size_t)n->info.width * (size_t)n->info.height);
  if (b2s_status st = b2s_hector_slam_copy_level_ros(n->proc, 0, n->payload.data())) return st;
  const int32_t rebuilt = map_gate(n, n->updates);
  if (on_map) on_map(user, (int32_t)n->scans, stamp, &n->info, n->payload.data(), rebuilt);
  return B2S_OK;
}

}  // extern "C"
