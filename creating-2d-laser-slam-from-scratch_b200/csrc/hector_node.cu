// lesson4's HectorMappingRos node (lesson4/src/hector_mapping/hector_slam.cc) over whole recordings, B nodes per handle:
// host C++ around the device fleet of HectorSlamProcessors (hector_slam.cu), one processor per node with its own map
// settings, whose ingest kernel k_hs_stream_batch<true, true> converts (hector_scan.cuh, with each node's own laser and
// filter) and matches every node's scans, one CTA per node.  The publish schedule and the launch parts are hector_node_plan.cuh's; the single-node entry points
// are the batched ones with B = 1.
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
#include <map>
#include <new>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "hector_node_plan.cuh"
#include "hector_scan.cuh"
#include "ros_math.cuh"

namespace b2s {
// hector_slam.cu
void hs_node_map_info(const b2s_hector_slam *p, int b, float &origin_x, float &origin_y, float &cell_length, int &w, int &h);
float hs_scale_to_map(const b2s_hector_slam *p, int b);
const char *hs_spec_error(const b2s_hector_map_spec &s);
b2s_hector_map_spec hs_default_spec(float map_resolution, int map_size_x, int map_size_y, float start_x, float start_y,
                                    int levels);
b2s_status hs_node_run(b2s_hector_slam *p, HsNodeIo &io, const HsLaser *lasers, const double *units, size_t n_units,
                       const HectorNodePlan &plan, const int32_t *n_scans, const float *ranges, float *out_rows,
                       const std::function<b2s_status(int, int, const int8_t *, const float *, long long)> &on_map);
}  // namespace b2s

using namespace b2s;

namespace {
constexpr int NODE_MAX_RANGES = 4096;      // the processor's per-scan capacity
constexpr int NODE_MAX_SCANS = (1 << 20) - 1;  // stamp epochs of one call (hector_slam.cu)
constexpr int NODE_MAX_BATCH = 65535;      // the publishes before one part are one launch's grid rows
constexpr int64_t NS = 1000000000LL;
}  // namespace

// B nodes, one per processor of a batched HectorSlamProcessor; per-node state is indexed by node
struct b2s_hector_node {
  int batch = 1;
  int device = 0;
  b2s_hector_slam *proc = nullptr;
  std::vector<HsLaser> lasers;  // node b's laser and filter (base: set per call)
  std::vector<double> units;    // the unit vectors of every distinct geometry ([n][2] each; HsLaser::unit0)
  std::vector<int64_t> period_ns;       // Duration::fromSec(map_pub_period)
  std::vector<HectorNodeClock> clock;   // the publish schedule (started, next tick)
  std::vector<int64_t> scans;           // scans handed in so far
  std::vector<int64_t> updates;         // map updates so far: level 0's getUpdateIndex() = updates - 1
  std::vector<int64_t> last_get_map_update_index;  // lastGetMapUpdateIndex
  std::vector<b2s_hector_node_map_info> info;  // node b's setMapInfo
  HsNodeIo io;
  std::vector<float> rows;
  std::vector<int8_t> payload;      // b2s_hector_node_publish_map_of's
  bool failed = false;              // a call failed partway: maps were handed out, the schedule was not committed
};

namespace {

// publishMap's gate: rebuild when node b's grid update index moved since its last publish
int32_t map_gate(b2s_hector_node *n, int b, int64_t updates) {
  const int64_t index = updates - 1;
  const bool rebuilt = index != n->last_get_map_update_index[(size_t)b];
  n->last_get_map_update_index[(size_t)b] = index;
  return rebuilt ? 1 : 0;
}

// the processor's fields (b2s_hector_node_create_batch requires them equal in every node's parameters)
bool same_processor(const b2s_hector_node_params &a, const b2s_hector_node_params &b) {
  return a.map_resolution == b.map_resolution && a.map_size == b.map_size &&
         a.map_multi_res_levels == b.map_multi_res_levels && a.map_start_x == b.map_start_x &&
         a.map_start_y == b.map_start_y && a.update_factor_free == b.update_factor_free &&
         a.update_factor_occupied == b.update_factor_occupied &&
         a.map_update_distance_thresh == b.map_update_distance_thresh &&
         a.map_update_angle_thresh == b.map_update_angle_thresh;
}

// a single-node entry point's callback behind the batched one
struct SingleMapFn {
  b2s_hector_node_map_fn fn;
  void *user;
};
void single_map(void *user, int32_t, int32_t scan_index, const uint32_t stamp[2], const b2s_hector_node_map_info *info,
                const int8_t *payload, int32_t rebuilt) {
  const SingleMapFn *s = static_cast<const SingleMapFn *>(user);
  if (s->fn) s->fn(s->user, scan_index, stamp, info, payload, rebuilt);
}

// Node b's processor: HectorSlamProcessor(static_cast<float>(resolution), size, size, Vector2f(start), levels) + the
// setters of the constructor
b2s_hector_map_spec node_spec(const b2s_hector_node_params &p) {
  b2s_hector_map_spec s = hs_default_spec(static_cast<float>(p.map_resolution), p.map_size, p.map_size,
                                          static_cast<float>(p.map_start_x), static_cast<float>(p.map_start_y),
                                          p.map_multi_res_levels);
  s.update_free = static_cast<float>(p.update_factor_free);
  s.update_occupied = static_cast<float>(p.update_factor_occupied);
  s.min_dist = static_cast<float>(p.map_update_distance_thresh);
  s.min_angle = static_cast<float>(p.map_update_angle_thresh);
  return s;
}

// The fleet behind every create entry point: node b's geometry is geometries[b * geometry_stride] (stride 0: one
// geometry for all).  `api` names the entry point in refusals, with the node when there are several.
b2s_status node_create(int batch, const b2s_hector_node_params *params, const b2s_laser_scan_msg *geometries,
                       int geometry_stride, const double *laser_mounts, int device, b2s_hector_node **out,
                       const char *api) {
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": null argument");
  *out = nullptr;
  if (!params || !geometries || !laser_mounts) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": null argument");
  if (batch < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": batch must be positive");
  if (batch > NODE_MAX_BATCH) B2S_FAIL(B2S_ERR_TOO_LARGE, std::string(api) + ": at most 65535 nodes");
  auto who = [&](int b) {
    return batch > 1 ? std::string(api) + ": node " + std::to_string(b) + ": " : std::string(api) + ": ";
  };
  std::vector<int64_t> period_ns((size_t)batch);
  std::vector<b2s_hector_map_spec> specs((size_t)batch);
  int most_ranges = 1;
  for (int b = 0; b < batch; b++) {
    const b2s_hector_node_params &pb = params[b];
    const b2s_laser_scan_msg &g = geometries[(size_t)b * geometry_stride];
    const double *mount = laser_mounts + 7 * (size_t)b;
    const float res = static_cast<float>(pb.map_resolution);
    if (!(res > 0.0f) || !std::isfinite(res)) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "map_resolution must be positive");
    if (pb.map_size <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "map_size must be positive");
    specs[(size_t)b] = node_spec(pb);
    if (const char *e = hs_spec_error(specs[(size_t)b])) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + e);
    const double period = pb.map_pub_period;
    if (!(period > 0.0) || !std::isfinite(period) || std::floor(period) > 2147483647.0)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "map_pub_period must be positive, finite and inside ros::Duration's range");
    const RosDuration d = ros_duration_from_sec(period);
    period_ns[(size_t)b] = (int64_t)d.sec * NS + (int64_t)d.nsec;
    if (period_ns[(size_t)b] <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "map_pub_period rounds to a zero ros::Duration");
    double qn = 0.0;
    for (int k = 0; k < 7; k++)
      if (!std::isfinite(mount[k])) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "non-finite laser mount");
    for (int k = 3; k < 7; k++) qn += mount[k] * mount[k];
    if (!(qn > 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "zero mount quaternion");
    if (g.angle_increment == 0.0f || g.n_ranges < 0)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "zero angle_increment or negative n_ranges");
    if (g.n_ranges > NODE_MAX_RANGES) B2S_FAIL(B2S_ERR_TOO_LARGE, who(b) + "at most 4096 ranges per scan");
    most_ranges = std::max(most_ranges, (int)g.n_ranges);
  }

  b2s_hector_slam *proc = nullptr;
  if (b2s_status st = b2s_hector_slam_create_fleet(batch, most_ranges, specs.data(), device, nullptr, &proc)) return st;
  b2s_hector_node *n = new (std::nothrow) b2s_hector_node();
  if (!n) {
    b2s_hector_slam_destroy(proc);
    B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  }
  std::unique_ptr<b2s_hector_node, decltype(&b2s_hector_node_destroy)> guard(n, b2s_hector_node_destroy);
  n->batch = batch;
  n->device = device;
  n->proc = proc;
  n->period_ns = period_ns;
  n->clock.assign((size_t)batch, HectorNodeClock{});
  n->scans.assign((size_t)batch, 0);
  n->updates.assign((size_t)batch, 0);
  n->last_get_map_update_index.assign((size_t)batch, -100);
  n->lasers.resize((size_t)batch);
  n->info.resize((size_t)batch);
  // every distinct geometry's unit vectors once: (angle_min, angle_increment, n_ranges) bits -> unit0
  std::map<std::tuple<uint32_t, uint32_t, int>, int> unit0;
  for (int b = 0; b < batch; b++) {
    const b2s_hector_node_params &pb = params[b];
    const b2s_laser_scan_msg &g = geometries[(size_t)b * geometry_stride];
    const double *mount = laser_mounts + 7 * (size_t)b;
    HsLaser &l = n->lasers[(size_t)b];
    std::memset(&l, 0, sizeof(l));
    // rosPointCloudToDataContainer's settings: the thresholds as InitParams stores them, the mount's tf::Transform
    HectorBeamFilter &f = l.filter;
    f.sqr_min = static_cast<float>(pb.laser_min_dist * pb.laser_min_dist);
    f.sqr_max = static_cast<float>(pb.laser_max_dist * pb.laser_max_dist);
    f.use_max_scan_range = pb.use_max_scan_range;
    tf_set_rotation(f.mount, mount + 3);
    f.mount.o[0] = mount[0]; f.mount.o[1] = mount[1]; f.mount.o[2] = mount[2];
    f.z_min = pb.laser_z_min_value;
    f.z_max = pb.laser_z_max_value;
    f.scale_to_map = hs_scale_to_map(proc, b);
    l.n_ranges = g.n_ranges;
    l.range_min = g.range_min;
    l.range_cutoff = 30.0;  // projector_.projectLaser(scan, laser_point_cloud_, 30.0)
    uint32_t am, ai;
    std::memcpy(&am, &g.angle_min, 4);
    std::memcpy(&ai, &g.angle_increment, 4);
    const auto key = std::make_tuple(am, ai, (int)g.n_ranges);
    auto it = unit0.find(key);
    if (it == unit0.end()) {
      it = unit0.emplace(key, (int)(n->units.size() / 2)).first;
      n->units.resize(n->units.size() + 2 * (size_t)g.n_ranges);
      hector_unit_vectors(g.angle_min, g.angle_increment, g.n_ranges, n->units.data() + 2 * (size_t)it->second);
    }
    l.unit0 = it->second;
    float ox, oy, cl;
    int w, h;
    hs_node_map_info(proc, b, ox, oy, cl, w, h);
    b2s_hector_node_map_info &info = n->info[(size_t)b];
    info.origin_x = ox; info.origin_y = oy;
    info.resolution = cl;
    info.width = w; info.height = h;
  }
  B2S_CUDA_CHECK(cudaSetDevice(device));
  B2S_CUDA_CHECK(n->io.copy.init(nullptr));
  for (int k = 0; k < 2; k++) {
    B2S_CUDA_CHECK(n->io.converted[k].create(cudaEventDisableTiming));
    B2S_CUDA_CHECK(n->io.copied[k].create(cudaEventDisableTiming));
  }
  *out = guard.release();
  return B2S_OK;
}

}  // namespace

extern "C" {

b2s_status b2s_hector_node_create_fleet(int batch, const b2s_hector_node_params *params,
                                        const b2s_laser_scan_msg *geometries, const double *laser_mounts, int device,
                                        b2s_hector_node **out) {
  return node_create(batch, params, geometries, 1, laser_mounts, device, out, "b2s_hector_node_create_fleet");
}

// the fleet with one geometry repeated, and the processor fields required equal
b2s_status b2s_hector_node_create_batch(int batch, const b2s_hector_node_params *params,
                                        const b2s_laser_scan_msg *geometry, const double *laser_mounts, int device,
                                        b2s_hector_node **out) {
  const char *api = batch == 1 ? "b2s_hector_node_create" : "b2s_hector_node_create_batch";
  if (out && params && batch > 1 && batch <= NODE_MAX_BATCH)
    for (int b = 1; b < batch; b++)
      if (!same_processor(params[b], params[0])) {
        *out = nullptr;
        B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": node " + std::to_string(b) +
                                         ": the processor's fields (map size, resolution, levels, start, update "
                                         "factors, update thresholds) differ from node 0's");
      }
  return node_create(batch, params, geometry, 0, laser_mounts, device, out, api);
}

b2s_status b2s_hector_node_create(const b2s_hector_node_params *params, const b2s_laser_scan_msg *geometry,
                                  const double laser_mount[7], int device, b2s_hector_node **out) {
  return b2s_hector_node_create_batch(1, params, geometry, laser_mount, device, out);
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

b2s_status b2s_hector_node_process_batch(b2s_hector_node *n, const int32_t *n_scans, const float *ranges,
                                         const uint32_t *stamps, float *out_pose, double *out_pose_msg, double *out_cov,
                                         int32_t *out_map_updated, int32_t *out_n_points,
                                         b2s_hector_node_batch_map_fn on_map, void *user) {
  B2S_NVTX("HectorMappingRos::scanCallback");
  if (!n || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_process: null argument");
  const int B = n->batch;
  size_t T = 0, floats = 0;
  bool too_many = false;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_process: negative scan count");
    T += (size_t)n_scans[b];
    floats += (size_t)n_scans[b] * (size_t)n->lasers[(size_t)b].n_ranges;
    too_many = too_many || n_scans[b] >= NODE_MAX_SCANS;
  }
  if (T > 0 && (!stamps || (!ranges && floats > 0)))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_process: null argument");
  if (n->failed) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_node_process: an earlier call failed partway; destroy the handle");
  if (too_many) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_hector_node_process: too many scans of one node in one call (split it)");
  if (T == 0) return B2S_OK;
  const HectorNodePlan plan = hector_node_plan(B, n_scans, stamps, n->clock.data(), n->period_ns.data());
  n->rows.resize(16 * T);
  std::vector<int64_t> updates = n->updates;  // node b's, through the rows handed to `publish` so far
  auto publish = [&](int b, int k, const int8_t *payload, const float *rows, long long n_rows) -> b2s_status {
    for (long long i = 0; i < n_rows; i++) updates[(size_t)b] += rows[16 * (size_t)i + 12] != 0.0f ? 1 : 0;
    const int32_t rebuilt = map_gate(n, b, updates[(size_t)b]);
    const int64_t tick = plan.ticks[(size_t)b][(size_t)k - 1];
    const uint32_t stamp[2] = {(uint32_t)(tick / NS), (uint32_t)(tick % NS)};
    if (on_map) on_map(user, b, (int32_t)(n->scans[(size_t)b] + plan.cuts[(size_t)b][(size_t)k - 1]), stamp,
                       &n->info[(size_t)b], payload, rebuilt);
    return B2S_OK;
  };
  b2s_status st = hs_node_run(n->proc, n->io, n->lasers.data(), n->units.data(), n->units.size() / 2, plan, n_scans,
                              ranges, n->rows.data(), publish);
  if (st) {
    // the processors, the maps handed out and the publish gates have moved, the schedules and the counters have not
    n->failed = true;
    return st;
  }
  n->clock = plan.after;
  size_t i = 0;
  for (int b = 0; b < B; b++) {
    for (int j = 0; j < n_scans[b]; j++, i++) {
      const float *r = n->rows.data() + 16 * i;
      const bool upd = r[12] != 0.0f;
      n->updates[(size_t)b] += upd ? 1 : 0;
      if (out_pose) std::memcpy(out_pose + 3 * i, r, 3 * sizeof(float));
      if (out_pose_msg) {
        // PoseInfoContainer::update: position x / y, orientation w = cos(yaw * 0.5f), z = sin(yaw * 0.5f) (double calls)
        double *m = out_pose_msg + 7 * i;
        const float half = r[2] * 0.5f;
        m[0] = (double)r[0]; m[1] = (double)r[1]; m[2] = 0.0;
        m[3] = 0.0; m[4] = 0.0; m[5] = sin((double)half); m[6] = cos((double)half);
      }
      if (out_cov) {
        const float *h = r + 3;  // row-major 3x3
        double *c = out_cov + 36 * i;
        for (int q = 0; q < 36; q++) c[q] = 0.0;
        c[0] = (double)h[0]; c[7] = (double)h[4]; c[35] = (double)h[8];
        c[1] = c[6] = (double)h[1];
        c[5] = c[30] = (double)h[2];
        c[11] = c[31] = (double)h[5];
      }
      if (out_map_updated) out_map_updated[i] = upd ? 1 : 0;
      if (out_n_points) std::memcpy(out_n_points + i, r + 15, sizeof(int32_t));
    }
    n->scans[(size_t)b] += n_scans[b];
  }
  return B2S_OK;
}

b2s_status b2s_hector_node_process(b2s_hector_node *n, int n_scans, const float *ranges, const uint32_t *stamps,
                                   float *out_pose, double *out_pose_msg, double *out_cov, int32_t *out_map_updated,
                                   int32_t *out_n_points, b2s_hector_node_map_fn on_map, void *user) {
  if (n && n->batch != 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_process: the handle has several nodes");
  const int32_t count = n_scans;
  SingleMapFn fn{on_map, user};
  return b2s_hector_node_process_batch(n, &count, ranges, stamps, out_pose, out_pose_msg, out_cov, out_map_updated,
                                       out_n_points, single_map, &fn);
}

b2s_status b2s_hector_node_publish_map_of(b2s_hector_node *n, int b, const uint32_t stamp[2],
                                          b2s_hector_node_batch_map_fn on_map, void *user) {
  if (!n || !stamp) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_publish_map: null argument");
  if (b < 0 || b >= n->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_publish_map_of: node index out of range");
  if (n->failed) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_node_publish_map: an earlier call failed partway; destroy the handle");
  const b2s_hector_node_map_info &info = n->info[(size_t)b];
  n->payload.resize((size_t)info.width * (size_t)info.height);
  if (b2s_status st = b2s_hector_slam_copy_level_ros_of(n->proc, b, 0, n->payload.data())) return st;
  const int32_t rebuilt = map_gate(n, b, n->updates[(size_t)b]);
  if (on_map) on_map(user, b, (int32_t)n->scans[(size_t)b], stamp, &info, n->payload.data(), rebuilt);
  return B2S_OK;
}

b2s_status b2s_hector_node_publish_map(b2s_hector_node *n, const uint32_t stamp[2], b2s_hector_node_map_fn on_map,
                                       void *user) {
  if (n && n->batch != 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_node_publish_map: the handle has several nodes");
  SingleMapFn fn{on_map, user};
  return b2s_hector_node_publish_map_of(n, 0, stamp, single_map, &fn);
}

}  // extern "C"
