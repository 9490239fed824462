// lesson6's SlamKarto node (lesson6/src/karto_slam.cc) over a whole recording of one laser: host C++ that drives the
// device Mapper (karto_mapper.cu, every MatchScan on the device) and the device occupancy grid (karto_occgrid.cu).
//   SlamKarto::InitParams / constructor              karto_slam.cc:21-58, 81-252
//   SlamKarto::laserCallback                         :286-325  (throttle, map-update gate)
//   SlamKarto::getLaser                              :327-405  (offset, upside-down test)
//   SlamKarto::addScan                               :407-481  (readings, Mapper::Process, map_to_odom_)
//   SlamKarto::getOdomPose                           :483-505
//   SlamKarto::updateMap                             :507-581  (CreateFromScans over every processed scan)
// tf's LinearMath and roscpp's Time / Duration are ros_math.cuh's (include/b200slam.h, DESIGN.md §7).
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "ros_math.cuh"

namespace b2s {
b2s_status karto_laser_from_msg(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                                b2s_laser *out);  // ros_io.cu
}

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

struct b2s_karto_node {
  b2s_karto_node_params prm{};
  b2s_laser laser{};
  int n_msg = 0, device = 0;
  bool inverted = false;
  TfTransform base_laser;
  RosDuration interval{0, 0};
  b2s_mapper *mapper = nullptr;
  int64_t laser_count = 0;  // laser_count_ (every scan handed in)
  bool got_map = false;
  uint32_t last_map_sec = 0, last_map_nsec = 0;  // laserCallback's static last_map_update
  double map_to_odom[7] = {0, 0, 0, 0, 0, 0, 1};
  bool failed = false;
  std::vector<double> readings;  // [processed scans][m], appended once per processed scan
  std::vector<double> poses;     // scratch for b2s_mapper_get_poses
  std::vector<double> scan;      // one scan's readings
  std::vector<int8_t> payload;   // scratch for b2s_occ_grid_copy_ros
};

namespace {

// SlamKarto::updateMap: CreateFromScans over every processed scan at its corrected pose now, then the ROS payload
b2s_status update_map(b2s_karto_node *n, int32_t scan_index, b2s_karto_map_fn on_map, void *user, bool &published) {
  published = false;
  const int count = b2s_mapper_scan_count(n->mapper);
  n->poses.resize(3 * (size_t)count);
  if (count > 0)
    if (b2s_status st = b2s_mapper_get_poses(n->mapper, n->poses.data())) return st;
  b2s_occ_grid *g = nullptr;
  if (b2s_status st = b2s_occ_grid_create_from_scans(&n->laser, count, n->readings.data(), n->poses.data(),
                                                     n->prm.resolution, n->device, nullptr, &g))
    return st;
  if (!g) return B2S_OK;  // CreateFromScans returned NULL: no map, the gate stays open
  b2s_occ_grid_info info;
  b2s_status st = b2s_occ_grid_info_get(g, &info);
  if (!st) {
    n->payload.resize((size_t)info.width * (size_t)info.height);
    st = b2s_occ_grid_copy_ros(g, n->payload.data());
  }
  b2s_occ_grid_destroy(g);
  if (st) return st;
  if (on_map) on_map(user, scan_index, &info, n->payload.data());
  published = true;
  return B2S_OK;
}

}  // namespace

extern "C" {

b2s_status b2s_karto_node_create(const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                                 const double laser_mount[7], const b2s_scan_solver *solver, int device,
                                 b2s_karto_node **out) {
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: null argument");
  *out = nullptr;
  if (!params || !geometry || !laser_mount) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: null argument");
  if (params->throttle_scans <= 0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: throttle_scans must be positive (the node divides by it)");
  if (!(params->resolution > 0.0) || !std::isfinite(params->resolution))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: resolution must be positive and finite");
  const double iv = params->map_update_interval;
  if (!std::isfinite(iv) || std::floor(iv) < -2147483648.0 || std::floor(iv) > 2147483647.0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: map_update_interval outside ros::Duration's range");
  double qn = 0.0;
  for (int k = 0; k < 7; k++)
    if (!std::isfinite(laser_mount[k])) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: non-finite laser mount");
  for (int k = 3; k < 7; k++) qn += laser_mount[k] * laser_mount[k];
  if (!(qn > 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: zero mount quaternion");

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
  if (b2s_status st = karto_laser_from_msg(geometry, offset, params->use_scan_range, &laser)) return st;
  if (laser.n_readings < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: the laser has no readings");
  if (geometry->n_ranges < laser.n_readings)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_create: the LaserScan carries fewer ranges than Round((angle_max - "
                                 "angle_min) / angle_increment); the node would read past them");

  b2s_mapper_params mp = params->mapper;
  mp.sequential.range_threshold = laser.range_threshold;  // Mapper::Initialize takes the laser's (Mapper.cpp)
  mp.loop.range_threshold = laser.range_threshold;
  b2s_mapper *mapper = nullptr;
  if (b2s_status st = b2s_mapper_create(&mp, &laser, device, &mapper)) return st;
  if (solver) {
    if (b2s_status st = b2s_mapper_set_scan_solver(mapper, solver)) {
      b2s_mapper_destroy(mapper);
      return st;
    }
  }
  b2s_karto_node *n = new (std::nothrow) b2s_karto_node();
  if (!n) {
    b2s_mapper_destroy(mapper);
    B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  }
  n->prm = *params;
  n->laser = laser;
  n->n_msg = geometry->n_ranges;
  n->device = device;
  n->inverted = up[2] <= 0;
  n->base_laser = base_laser;
  n->interval = ros_duration_from_sec(iv);
  n->mapper = mapper;
  n->scan.resize((size_t)laser.n_readings);
  *out = n;
  return B2S_OK;
}

void b2s_karto_node_destroy(b2s_karto_node *n) {
  if (!n) return;
  b2s_mapper_destroy(n->mapper);
  delete n;
}

b2s_mapper *b2s_karto_node_mapper(b2s_karto_node *n) { return n ? n->mapper : nullptr; }

b2s_status b2s_karto_node_process(b2s_karto_node *n, int n_scans, const float *ranges, const uint32_t *stamps,
                                  const double *odom, int32_t *out_state, double *out_pose, double *out_map_to_odom,
                                  int32_t *out_map_published, b2s_karto_map_fn on_map, void *user) {
  B2S_NVTX("SlamKarto::laserCallback");
  if (!n || n_scans < 0 || (n_scans > 0 && (!ranges || !stamps || !odom)))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_karto_node_process: null argument or negative count");
  if (n->failed)
    B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_karto_node_process: an earlier call failed inside the Mapper; destroy the handle");
  const int m = n->laser.n_readings, nr = n->n_msg;
  for (int i = 0; i < n_scans; i++) {
    const int32_t scan_index = (int32_t)n->laser_count;
    int32_t state = B2S_KARTO_THROTTLED, published = 0;
    double pose[3] = {0, 0, 0};
    n->laser_count++;
    if (n->laser_count % n->prm.throttle_scans == 0) {
      // getOdomPose: transformPose(odom_frame_, identity in base_frame_) at the scan's stamp
      const double *row = odom + 7 * (size_t)i;
      bool ok = true;
      for (int k = 0; k < 7; k++) ok = ok && !std::isnan(row[k]);
      if (!ok) {
        state = B2S_KARTO_NO_ODOM;
      } else {
        const TfTransform odom_base = tf_from_row(row);
        double ident[7] = {0, 0, 0};  // tf::Transform(createQuaternionFromRPY(0, 0, 0), (0, 0, 0))
        quat_set_rpy(0, 0, 0, ident + 3);
        const TfTransform op = tf_mul(odom_base, tf_from_row(ident));
        const double odom_pose[3] = {op.o[0], op.o[1], yaw_of(op)};
        // addScan: float32 ranges widened, reversed for an upside-down laser; the laser's m readings are used
        const float *r = ranges + (size_t)i * nr;
        for (int k = 0; k < m; k++) n->scan[k] = (double)r[n->inverted ? nr - 1 - k : k];
        int32_t processed = 0;
        b2s_status st = b2s_mapper_process_sensor(n->mapper, "laser", n->scan.data(), odom_pose, 0.0, &processed, pose);
        if (st) {
          n->failed = true;
          return st;
        }
        if (!processed) {
          state = B2S_KARTO_NOT_MOVED;
          pose[0] = pose[1] = pose[2] = 0;
        } else {
          state = B2S_KARTO_PROCESSED;
          n->readings.insert(n->readings.end(), n->scan.begin(), n->scan.end());
          // map_to_odom_ = (odom <- base_link * T(corrected)^-1) rebuilt from its quaternion and origin, inverted
          double corrected[7] = {pose[0], pose[1], 0.0}, odom_to_map[7];
          quat_set_rpy(0, 0, pose[2], corrected + 3);
          tf_to_row(tf_mul(odom_base, tf_inverse(tf_from_row(corrected))), odom_to_map);
          tf_to_row(tf_inverse(tf_from_row(odom_to_map)), n->map_to_odom);
          const uint32_t *s = stamps + 2 * (size_t)i;
          if (!n->got_map || ros_duration_gt(ros_time_diff(s[0], s[1], n->last_map_sec, n->last_map_nsec), n->interval)) {
            bool done = false;
            if ((st = update_map(n, scan_index, on_map, user, done))) {
              n->failed = true;
              return st;
            }
            if (done) {
              n->last_map_sec = s[0];
              n->last_map_nsec = s[1];
              n->got_map = true;
              published = 1;
            }
          }
        }
      }
    }
    if (out_state) out_state[i] = state;
    if (out_pose) std::memcpy(out_pose + 3 * (size_t)i, pose, sizeof pose);
    if (out_map_to_odom) std::memcpy(out_map_to_odom + 7 * (size_t)i, n->map_to_odom, sizeof n->map_to_odom);
    if (out_map_published) out_map_published[i] = published;
  }
  return B2S_OK;
}

}  // extern "C"
