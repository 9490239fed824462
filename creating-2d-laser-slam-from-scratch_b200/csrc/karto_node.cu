// lesson6's SlamKarto node (lesson6/src/karto_slam.cc) over whole recordings, B nodes per handle: host C++ that drives
// one Mapper per node (karto_mapper.cu) and the device occupancy grid (karto_occgrid.cu).  Each node runs its per-scan
// loop, unchanged, on a worker thread of its own; its device work (every MatchScan batch, every map build) becomes a
// request to the dispatcher on the calling thread, which serves the requests of all nodes in rounds: the matches on
// one MatchPool (karto_mapper.cu) whose every client is a node, the maps in one batched build.  The single-node handle
// is the batch of one.
//   SlamKarto::InitParams / constructor              karto_slam.cc:21-58, 81-252
//   SlamKarto::laserCallback                         :286-325  (throttle, map-update gate)
//   SlamKarto::getLaser                              :327-405  (offset, upside-down test)
//   SlamKarto::addScan                               :407-481  (readings, Mapper::Process, map_to_odom_)
//   SlamKarto::getOdomPose                           :483-505
//   SlamKarto::updateMap                             :507-581  (CreateFromScans over every processed scan)
// tf's LinearMath and roscpp's Time / Duration are ros_math.cuh's (include/b200slam.h, DESIGN.md §7).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstddef>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"
#include "karto_internal.cuh"
#include "ros_math.cuh"

using namespace b2s;

namespace {

// tf::Transform(q, origin) from a row (x, y, z, qx, qy, qz, qw)
TfTransform tf_from_row(const double *r) {
  TfTransform t;
  tf_set_rotation(t, r + 3);
  t.o[0] = r[0]; t.o[1] = r[1]; t.o[2] = r[2];
  return t;
}

void tf_to_row(const TfTransform &t, double *out) {
  out[0] = t.o[0]; out[1] = t.o[1]; out[2] = t.o[2];
  tf_get_rotation(t, out + 3);
}

// tf::getYaw(transform.getRotation())
double yaw_of(const TfTransform &t) {
  double q[4];
  tf_get_rotation(t, q);
  return tf_get_yaw(q);
}

}  // namespace

namespace {

constexpr int NODE_MAX_BATCH = 1024;  // nodes per handle

// a node's device work, posted by its worker and served by the dispatcher
struct Request {
  const MatchRequest *match = nullptr;  // a MatchScan batch, or else a map build
  // a map build: CreateFromScans over the node's first `count` scans at `map_poses`
  int32_t scan_index = 0, count = 0;
  const double *map_poses = nullptr;
  int32_t published = 0;  // out: a map was built and handed to on_map
  b2s_status status = B2S_OK;
  bool done = false;
};

struct Failure {
  long long round = -1;  // the round before which it happened
  int node = -1;
  b2s_status status = B2S_OK;
  std::string message;
  bool before(const Failure &o) const { return o.node < 0 || round < o.round || (round == o.round && node < o.node); }
};

// one call's rendezvous of the workers and the dispatcher: a round is served when every worker that has not finished
// has posted its next request, so round k holds each live node's k-th request whatever the thread timing
struct Lockstep {
  std::mutex mu;
  std::condition_variable to_dispatcher, to_workers;
  int live = 0, waiting = 0;
  long long round = 0;
  std::vector<Request *> posted;  // [batch]
  Failure first;
  bool stop = false;              // a failure was recorded: every later request is refused
  void fail(const Failure &f) {
    if (f.before(first)) first = f;
    stop = true;
  }
};

}  // namespace

// one SlamKarto of a handle
struct KartoNodeState {
  b2s_karto_node *owner = nullptr;
  int index = 0;
  b2s_karto_node_params prm{};
  RosDuration interval{0, 0};
  b2s_mapper *mapper = nullptr;
  int64_t laser_count = 0;  // laser_count_ (every scan handed in)
  bool got_map = false;
  uint32_t last_map_sec = 0, last_map_nsec = 0;  // laserCallback's static last_map_update
  double map_to_odom[7] = {0, 0, 0, 0, 0, 0, 1};
  std::vector<double> scan;                      // one scan's readings
  std::vector<double> poses;                     // scratch for b2s_mapper_get_poses
  std::vector<int32_t> map_row;                  // row in the map pool of each Mapper scan
};

struct b2s_karto_node {
  int batch = 1;
  b2s_laser laser{};
  int n_msg = 0, device = 0;
  bool inverted = false;
  b2s_matcher_params matcher_params[2]{};
  std::vector<KartoNodeState> nodes;
  MatchPool *matches = nullptr;  // every node is a client, numbered by its index
  OccBatch *maps = nullptr;
  Lockstep *lock = nullptr;  // the running call's
  bool failed = false;
  double timing[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  std::vector<float> stage;  // the dispatcher's scratch
};

namespace {

// set on a worker whose request was refused or failed on the device: the dispatcher has recorded the failure
thread_local bool t_stopped = false;

// a worker's request: posted, then the worker waits until the dispatcher served it
b2s_status post(KartoNodeState &k, Request &r) {
  Lockstep &L = *k.owner->lock;
  std::unique_lock<std::mutex> g(L.mu);
  if (!L.stop) {
    L.posted[(size_t)k.index] = &r;
    L.waiting++;
    if (L.waiting == L.live) L.to_dispatcher.notify_one();
    L.to_workers.wait(g, [&] { return r.done; });
    if (!r.status) return B2S_OK;
  }
  t_stopped = true;
  B2S_FAIL(B2S_ERR_BAD_STATE, "stopped: a node of the handle failed");
}

// FleetMatchFn: the Mapper's match batch as a request
b2s_status fleet_match(void *user, const MatchRequest &m) {
  Request r;
  r.match = &m;
  return post(*static_cast<KartoNodeState *>(user), r);
}

// SlamKarto::updateMap as a request: CreateFromScans over every processed scan at its corrected pose now
b2s_status update_map(KartoNodeState &k, int32_t scan_index, bool &published) {
  published = false;
  const int count = b2s_mapper_scan_count(k.mapper);
  k.poses.resize(3 * (size_t)count);
  if (count > 0)
    if (b2s_status st = b2s_mapper_get_poses(k.mapper, k.poses.data())) return st;
  Request r;
  r.scan_index = scan_index;
  r.count = count;
  r.map_poses = k.poses.data();
  if (b2s_status st = post(k, r)) return st;
  published = r.published != 0;  // CreateFromScans returned NULL: no map, the gate stays open
  return B2S_OK;
}

struct CallRows {
  const float *ranges;
  const uint32_t *stamps;
  const double *odom;
  int32_t *out_state;
  double *out_pose, *out_map_to_odom;
  int32_t *out_map_published;
};

// SlamKarto::laserCallback on scan `i` of the call's rows (node-major), the body of the single node's loop
b2s_status node_scan(b2s_karto_node *n, KartoNodeState &k, size_t i, const CallRows &a) {
  const int m = n->laser.n_readings, nr = n->n_msg;
  const int32_t scan_index = (int32_t)k.laser_count;
  int32_t state = B2S_KARTO_THROTTLED, published = 0;
  double pose[3] = {0, 0, 0};
  k.laser_count++;
  if (k.laser_count % k.prm.throttle_scans == 0) {
    // getOdomPose: transformPose(odom_frame_, identity in base_frame_) at the scan's stamp
    const double *row = a.odom + 7 * i;
    bool ok = true;
    for (int q = 0; q < 7; q++) ok = ok && !std::isnan(row[q]);
    if (!ok) {
      state = B2S_KARTO_NO_ODOM;
    } else {
      const TfTransform odom_base = tf_from_row(row);
      double ident[7] = {0, 0, 0};  // tf::Transform(createQuaternionFromRPY(0, 0, 0), (0, 0, 0))
      quat_set_rpy(0, 0, 0, ident + 3);
      const TfTransform op = tf_mul(odom_base, tf_from_row(ident));
      const double odom_pose[3] = {op.o[0], op.o[1], yaw_of(op)};
      // addScan: float32 ranges widened, reversed for an upside-down laser; the laser's m readings are used
      const float *r = a.ranges + i * (size_t)nr;
      for (int q = 0; q < m; q++) k.scan[q] = (double)r[n->inverted ? nr - 1 - q : q];
      int32_t processed = 0;
      if (b2s_status st = b2s_mapper_process_sensor(k.mapper, "laser", k.scan.data(), odom_pose, 0.0, &processed, pose))
        return st;
      if (!processed) {
        state = B2S_KARTO_NOT_MOVED;
        pose[0] = pose[1] = pose[2] = 0;
      } else {
        state = B2S_KARTO_PROCESSED;
        // map_to_odom_ = (odom <- base_link * T(corrected)^-1) rebuilt from its quaternion and origin, inverted
        double corrected[7] = {pose[0], pose[1], 0.0}, odom_to_map[7];
        quat_set_rpy(0, 0, pose[2], corrected + 3);
        tf_to_row(tf_mul(odom_base, tf_inverse(tf_from_row(corrected))), odom_to_map);
        tf_to_row(tf_inverse(tf_from_row(odom_to_map)), k.map_to_odom);
        const uint32_t *s = a.stamps + 2 * i;
        if (!k.got_map || ros_duration_gt(ros_time_diff(s[0], s[1], k.last_map_sec, k.last_map_nsec), k.interval)) {
          bool done = false;
          if (b2s_status st = update_map(k, scan_index, done)) return st;
          if (done) {
            k.last_map_sec = s[0];
            k.last_map_nsec = s[1];
            k.got_map = true;
            published = 1;
          }
        }
      }
    }
  }
  if (a.out_state) a.out_state[i] = state;
  if (a.out_pose) std::memcpy(a.out_pose + 3 * i, pose, sizeof pose);
  if (a.out_map_to_odom) std::memcpy(a.out_map_to_odom + 7 * i, k.map_to_odom, sizeof k.map_to_odom);
  if (a.out_map_published) a.out_map_published[i] = published;
  return B2S_OK;
}

// a worker: node b's scans of the call, then it leaves the lockstep.  It makes no CUDA call and never calls on_map.
void worker(b2s_karto_node *n, int b, size_t first, int count, const CallRows &a) {
  KartoNodeState &k = n->nodes[(size_t)b];
  Lockstep &L = *n->lock;
  b2s_status st = B2S_OK;
  for (int i = 0; i < count && !st; i++) st = node_scan(n, k, first + (size_t)i, a);
  std::lock_guard<std::mutex> g(L.mu);
  if (st && !t_stopped) {
    Failure f;
    f.round = L.round;
    f.node = b;
    f.status = st;
    f.message = b2s_last_error();
    L.fail(f);
  }
  L.live--;
  if (L.waiting == L.live) L.to_dispatcher.notify_one();
}

// one group of match requests with the same (which, do_penalize, do_refine), node order, on the nodes' shared pool
b2s_status serve_matches(b2s_karto_node *n, const std::vector<std::pair<int, Request *>> &group) {
  std::vector<std::pair<int, const MatchRequest *>> reqs;
  for (const auto &q : group) reqs.emplace_back(q.first, q.second->match);
  return match_pool_serve(n->matches, reqs, &n->timing[1]);  // timing[1], [2]: match launches, matches
}

// every map request of a round in one batched build; maps to on_map in ascending node order
b2s_status serve_maps(b2s_karto_node *n, const std::vector<std::pair<int, Request *>> &reqs, b2s_karto_node_batch_map_fn on_map,
                      void *user) {
  const int G = (int)reqs.size(), m = n->laser.n_readings;
  // each node's scans not yet in the map pool, float32 (they are float32 ranges widened, so this is exact), one upload
  size_t fresh = 0;
  for (const auto &q : reqs) fresh += (size_t)q.second->count - std::min(n->nodes[(size_t)q.first].map_row.size(), (size_t)q.second->count);
  n->stage.resize(fresh * (size_t)m);
  size_t s = 0;
  for (const auto &q : reqs) {
    const KartoNodeState &k = n->nodes[(size_t)q.first];
    for (int id = (int)k.map_row.size(); id < q.second->count; id++, s++) {
      const double *r = mapper_scan_ranges(k.mapper, id);
      for (int i = 0; i < m; i++) n->stage[s * m + i] = (float)r[i];
    }
  }
  int32_t first = 0;
  if (b2s_status st = occ_batch_append(n->maps, (int)fresh, n->stage.data(), &first)) return st;
  std::vector<int32_t> n_scans((size_t)G), rows, have((size_t)G);
  std::vector<double> poses, res((size_t)G);
  for (int g = 0; g < G; g++) {
    KartoNodeState &k = n->nodes[(size_t)reqs[(size_t)g].first];
    const Request &r = *reqs[(size_t)g].second;
    while ((int)k.map_row.size() < r.count) k.map_row.push_back(first++);
    n_scans[(size_t)g] = r.count;
    rows.insert(rows.end(), k.map_row.begin(), k.map_row.begin() + r.count);
    poses.insert(poses.end(), r.map_poses, r.map_poses + 3 * (size_t)r.count);
    res[(size_t)g] = k.prm.resolution;
  }
  std::vector<b2s_occ_grid_info> info((size_t)G);
  std::vector<const int8_t *> payload((size_t)G);
  if (b2s_status st = occ_batch_build(n->maps, G, n_scans.data(), rows.data(), poses.data(), res.data(), info.data(),
                                      have.data(), payload.data()))
    return st;
  for (int g = 0; g < G; g++) {
    Request &r = *reqs[(size_t)g].second;
    if (!have[(size_t)g]) continue;
    if (on_map) on_map(user, reqs[(size_t)g].first, r.scan_index, &info[(size_t)g], payload[(size_t)g]);
    r.published = 1;
    n->timing[3] += 1;
  }
  return B2S_OK;
}

double seconds_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// one round: matches by group, then the maps; a failure stops every node at its next request
void serve_round(b2s_karto_node *n, Lockstep &L, const std::vector<std::pair<int, Request *>> &reqs,
                 b2s_karto_node_batch_map_fn on_map, void *user) {
  if (L.stop) {  // a worker failed since the last round
    for (const auto &q : reqs) q.second->status = B2S_ERR_BAD_STATE;
    return;
  }
  std::vector<std::pair<int, Request *>> maps;
  std::vector<std::vector<std::pair<int, Request *>>> groups;
  std::vector<int> keys;
  for (const auto &q : reqs) {
    const MatchRequest *m = q.second->match;
    if (!m) {
      maps.push_back(q);
      continue;
    }
    const int key = m->which * 4 + m->do_penalize * 2 + m->do_refine;
    size_t gi = 0;
    while (gi < keys.size() && keys[gi] != key) gi++;
    if (gi == keys.size()) {
      keys.push_back(key);
      groups.emplace_back();
    }
    groups[gi].push_back(q);
  }
  auto fail = [&](const std::vector<std::pair<int, Request *>> &g, b2s_status st) {
    Failure f;
    f.round = L.round;
    f.node = g[0].first;
    f.status = st;
    f.message = b2s_last_error();
    std::lock_guard<std::mutex> lk(L.mu);
    L.fail(f);
  };
  auto t0 = std::chrono::steady_clock::now();
  for (const auto &g : groups) {
    b2s_status st = L.stop ? B2S_ERR_BAD_STATE : serve_matches(n, g);
    if (st && !L.stop) fail(g, st);
    for (const auto &q : g) q.second->status = st;
  }
  n->timing[4] += seconds_since(t0);
  if (!maps.empty()) {
    t0 = std::chrono::steady_clock::now();
    b2s_status st = L.stop ? B2S_ERR_BAD_STATE : serve_maps(n, maps, on_map, user);
    if (st && !L.stop) fail(maps, st);
    for (const auto &q : maps) q.second->status = st;
    n->timing[5] += seconds_since(t0);
  }
}

// the fields a node's getLaser derives, equal bit for bit
bool same_bits(const void *a, const void *b, size_t n) { return std::memcmp(a, b, n) == 0; }
bool same_laser(const b2s_laser &a, const b2s_laser &b) {
  return a.n_readings == b.n_readings && same_bits(&a.min_angle, &b.min_angle, 8) &&
         same_bits(&a.angular_resolution, &b.angular_resolution, 8) && same_bits(&a.min_range, &b.min_range, 8) &&
         same_bits(&a.max_range, &b.max_range, 8) && same_bits(&a.range_threshold, &b.range_threshold, 8) &&
         same_bits(a.offset_pose, b.offset_pose, sizeof a.offset_pose);
}
bool same_matcher(const b2s_matcher_params &a, const b2s_matcher_params &b) {
  return same_bits(&a, &b, offsetof(b2s_matcher_params, use_response_expansion)) &&
         a.use_response_expansion == b.use_response_expansion;
}

// a single-node entry point's callback behind the batched one
struct SingleMapFn {
  b2s_karto_map_fn fn;
  void *user;
};
void single_map(void *user, int32_t, int32_t scan_index, const b2s_occ_grid_info *info, const int8_t *payload) {
  const SingleMapFn *s = static_cast<const SingleMapFn *>(user);
  if (s->fn) s->fn(s->user, scan_index, info, payload);
}

// the handle; `single`: b2s_karto_node_create's solver rule (any non-NULL solver is set), else a slot whose compute is
// NULL means no back end
b2s_status create_impl(int batch, const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                       const double *laser_mounts, const b2s_scan_solver *solvers, bool single, int device,
                       b2s_karto_node **out) {
  const char *fn = single ? "b2s_karto_node_create" : "b2s_karto_node_create_batch";
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(fn) + ": null argument");
  *out = nullptr;
  if (!params || !geometry || !laser_mounts) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(fn) + ": null argument");
  if (batch < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(fn) + ": batch must be positive");
  if (batch > NODE_MAX_BATCH) B2S_FAIL(B2S_ERR_TOO_LARGE, std::string(fn) + ": at most 1024 nodes");
  std::unique_ptr<b2s_karto_node, decltype(&b2s_karto_node_destroy)> n(new (std::nothrow) b2s_karto_node(),
                                                                      b2s_karto_node_destroy);
  if (!n) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  n->batch = batch;
  n->device = device;
  n->n_msg = geometry->n_ranges;
  n->nodes.resize((size_t)batch);
  int window = 0;  // the longest running window of the nodes
  for (int b = 0; b < batch; b++) {
    const b2s_karto_node_params *p = params + b;
    const double *laser_mount = laser_mounts + 7 * (size_t)b;
    const std::string who = single ? std::string("b2s_karto_node_create: ")
                                   : "b2s_karto_node_create_batch: node " + std::to_string(b) + ": ";
    if (p->throttle_scans <= 0)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "throttle_scans must be positive (the node divides by it)");
    if (!(p->resolution > 0.0) || !std::isfinite(p->resolution))
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "resolution must be positive and finite");
    const double iv = p->map_update_interval;
    if (!std::isfinite(iv) || std::floor(iv) < -2147483648.0 || std::floor(iv) > 2147483647.0)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "map_update_interval outside ros::Duration's range");
    double qn = 0.0;
    for (int k = 0; k < 7; k++)
      if (!std::isfinite(laser_mount[k])) B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "non-finite laser mount");
    for (int k = 3; k < 7; k++) qn += laser_mount[k] * laser_mount[k];
    if (!(qn > 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "zero mount quaternion");

    // getLaser: transformPose(base_frame_, identity in the laser frame), getYaw, and the upside-down test
    const TfTransform base_laser = tf_from_row(laser_mount);
    TfTransform identity;
    tf_identity(identity);
    const TfTransform laser_pose = tf_mul(base_laser, identity);
    const double offset[3] = {laser_pose.o[0], laser_pose.o[1], yaw_of(laser_pose)};
    const double up_in_laser[3] = {0, 0, 1 + laser_pose.o[2]};
    double up[3];
    tf_apply(tf_inverse(base_laser), up_in_laser, up);
    b2s_laser laser;
    if (b2s_status st = karto_laser_from_msg(geometry, offset, p->use_scan_range, &laser)) {
      if (!single) set_last_error(who + b2s_last_error());
      return st;
    }
    if (laser.n_readings < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "the laser has no readings");
    if (geometry->n_ranges < laser.n_readings)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "the LaserScan carries fewer ranges than Round((angle_max - angle_min) / "
                                         "angle_increment); the node would read past them");
    b2s_mapper_params mp = p->mapper;
    mp.sequential.range_threshold = laser.range_threshold;  // Mapper::Initialize takes the laser's (Mapper.cpp)
    mp.loop.range_threshold = laser.range_threshold;
    const bool inverted = up[2] <= 0;
    if (b == 0) {
      n->laser = laser;
      n->inverted = inverted;
      n->matcher_params[0] = mp.sequential;
      n->matcher_params[1] = mp.loop;
    } else {
      // every node shares the two matchers and the map kernels' laser
      if (!same_laser(laser, n->laser) || inverted != n->inverted)
        B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "its laser (offset, range threshold or upside-down flag) differs from node 0's");
      if (!same_matcher(mp.sequential, n->matcher_params[0]) || !same_matcher(mp.loop, n->matcher_params[1]))
        B2S_FAIL(B2S_ERR_BAD_PARAMS, who + "its matcher parameters (mapper.sequential / mapper.loop) differ from node 0's");
    }
    KartoNodeState &k = n->nodes[(size_t)b];
    k.owner = n.get();
    k.index = b;
    k.prm = *p;
    k.interval = ros_duration_from_sec(iv);
    k.scan.resize((size_t)laser.n_readings);
    if (b2s_status st = mapper_create_fleet(&mp, &laser, fleet_match, &k, &k.mapper)) {
      if (!single) set_last_error(who + b2s_last_error());
      return st;
    }
    const b2s_scan_solver *solver = solvers ? solvers + b : nullptr;
    if (solver && (single || solver->compute))
      if (b2s_status st = b2s_mapper_set_scan_solver(k.mapper, solver)) return st;
    window = std::max(window, p->mapper.scan_buffer_size);
  }
  if (b2s_status st = check_device(device)) return st;
  if (b2s_status st = match_pool_create(n->matcher_params, n->laser, device, batch, window, &n->matches)) return st;
  if (b2s_status st = occ_batch_create(n->laser, device, &n->maps)) return st;
  *out = n.release();
  return B2S_OK;
}

}  // namespace

extern "C" {

b2s_status b2s_karto_node_create_batch(int batch, const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                                       const double *laser_mounts, const b2s_scan_solver *solvers, int device,
                                       b2s_karto_node **out) {
  return create_impl(batch, params, geometry, laser_mounts, solvers, false, device, out);
}

b2s_status b2s_karto_node_create(const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                                 const double laser_mount[7], const b2s_scan_solver *solver, int device,
                                 b2s_karto_node **out) {
  return create_impl(1, params, geometry, laser_mount, solver, true, device, out);
}

void b2s_karto_node_destroy(b2s_karto_node *n) {
  if (!n) return;
  for (KartoNodeState &k : n->nodes) b2s_mapper_destroy(k.mapper);
  match_pool_destroy(n->matches);
  occ_batch_destroy(n->maps);
  delete n;
}

b2s_mapper *b2s_karto_node_mapper(b2s_karto_node *n) { return n && n->batch == 1 ? n->nodes[0].mapper : nullptr; }

b2s_mapper *b2s_karto_node_mapper_of(b2s_karto_node *n, int b) {
  return n && b >= 0 && b < n->batch ? n->nodes[(size_t)b].mapper : nullptr;
}

b2s_status b2s_karto_node_process_batch(b2s_karto_node *n, const int32_t *n_scans, const float *ranges,
                                        const uint32_t *stamps, const double *odom, int32_t *out_state, double *out_pose,
                                        double *out_map_to_odom, int32_t *out_map_published,
                                        b2s_karto_node_batch_map_fn on_map, void *user) {
  B2S_NVTX("SlamKarto::laserCallback");
  if (!n || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: null argument or negative count");
  const int B = n->batch;
  size_t T = 0;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: null argument or negative count");
    T += (size_t)n_scans[b];
  }
  if (T > 0 && (!ranges || !stamps || !odom))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: null argument or negative count");
  if (n->failed)
    B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_karto_node_process: an earlier call failed inside the Mapper; destroy the handle");
  for (double &t : n->timing) t = 0;
  if (T == 0) return B2S_OK;
  const auto t0 = std::chrono::steady_clock::now();
  const double bytes0 = occ_batch_bytes_d2h(n->maps);
  B2S_CUDA_CHECK(cudaSetDevice(n->device));
  const CallRows rows{ranges, stamps, odom, out_state, out_pose, out_map_to_odom, out_map_published};
  Lockstep L;
  L.posted.assign((size_t)B, nullptr);
  n->lock = &L;
  std::vector<std::thread> threads;
  threads.reserve((size_t)B);
  {
    std::lock_guard<std::mutex> g(L.mu);  // no worker posts before every worker is counted
    size_t first = 0;
    for (int b = 0; b < B; b++) {
      if (n_scans[b] > 0) {
        try {
          threads.emplace_back(worker, n, b, first, (int)n_scans[b], std::cref(rows));
          L.live++;
        } catch (...) {
          Failure f;
          f.round = 0;
          f.node = b;
          f.status = B2S_ERR_CUDA;
          f.message = "could not start a worker thread";
          L.fail(f);
          break;
        }
      }
      first += (size_t)n_scans[b];
    }
  }
  // the dispatcher
  std::vector<std::pair<int, Request *>> reqs;
  for (;;) {
    {
      std::unique_lock<std::mutex> g(L.mu);
      L.to_dispatcher.wait(g, [&] { return L.waiting == L.live; });
      if (L.live == 0) break;
      reqs.clear();
      for (int b = 0; b < B; b++)
        if (L.posted[(size_t)b]) reqs.emplace_back(b, L.posted[(size_t)b]);
    }
    serve_round(n, L, reqs, on_map, user);
    n->timing[0] += 1;
    {
      std::lock_guard<std::mutex> g(L.mu);
      for (auto &q : reqs) {
        q.second->done = true;
        L.posted[(size_t)q.first] = nullptr;
      }
      L.waiting = 0;
      L.round++;
    }
    L.to_workers.notify_all();
  }
  for (std::thread &t : threads) t.join();
  n->lock = nullptr;
  n->timing[6] = occ_batch_bytes_d2h(n->maps) - bytes0;
  n->timing[7] = seconds_since(t0);
  if (L.first.node >= 0) {
    // the Mappers, the maps handed out and the nodes' rows up to their stop have moved
    n->failed = true;
    set_last_error(B > 1 ? "b2s_karto_node_process_batch: node " + std::to_string(L.first.node) + ": " + L.first.message
                         : L.first.message);
    return L.first.status;
  }
  return B2S_OK;
}

b2s_status b2s_karto_node_process(b2s_karto_node *n, int n_scans, const float *ranges, const uint32_t *stamps,
                                  const double *odom, int32_t *out_state, double *out_pose, double *out_map_to_odom,
                                  int32_t *out_map_published, b2s_karto_map_fn on_map, void *user) {
  if (n && n->batch != 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: the handle has several nodes");
  if (n_scans < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: null argument or negative count");
  const int32_t count = n_scans;
  SingleMapFn fn{on_map, user};
  return b2s_karto_node_process_batch(n, &count, ranges, stamps, odom, out_state, out_pose, out_map_to_odom,
                                      out_map_published, single_map, &fn);
}

b2s_status b2s_karto_node_last_timing(const b2s_karto_node *n, double out[8]) {
  if (!n || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  std::memcpy(out, n->timing, sizeof n->timing);
  return B2S_OK;
}

}  // extern "C"
