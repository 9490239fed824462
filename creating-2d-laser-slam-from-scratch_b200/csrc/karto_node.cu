// lesson6's SlamKarto node (lesson6/src/karto_slam.cc) over a whole recording of one laser: host C++ that drives the
// device Mapper (karto_mapper.cu, every MatchScan on the device) and the device occupancy grid (karto_occgrid.cu).
//   SlamKarto::InitParams / constructor              karto_slam.cc:21-58, 81-252
//   SlamKarto::laserCallback                         :286-325  (throttle, map-update gate)
//   SlamKarto::getLaser                              :327-405  (offset, upside-down test)
//   SlamKarto::addScan                               :407-481  (readings, Mapper::Process, map_to_odom_)
//   SlamKarto::getOdomPose                           :483-505
//   SlamKarto::updateMap                             :507-581  (CreateFromScans over every processed scan)
// tf's LinearMath and roscpp's Time / Duration are restated below in double / integer arithmetic, operation by operation
// (include/b200slam.h, DESIGN.md §7).
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace b2s {
b2s_status karto_laser_from_msg(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                                b2s_laser *out);  // ros_io.cu
}

using namespace b2s;

namespace {

// ---- tf LinearMath (tf/LinearMath/{Vector3,Quaternion,Matrix3x3,Transform}.h), double, no FMA contraction
struct V3 {
  double x, y, z;
};
inline double dot(const V3 &a, const V3 &b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

struct Quat {
  double x, y, z, w;
};

struct M33 {
  V3 r[3];  // rows
  static M33 identity() { return M33{{{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}}; }
  // Matrix3x3::setRotation
  static M33 rotation(const Quat &q) {
    const double d = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    const double s = 2.0 / d;
    const double xs = q.x * s, ys = q.y * s, zs = q.z * s;
    const double wx = q.w * xs, wy = q.w * ys, wz = q.w * zs;
    const double xx = q.x * xs, xy = q.x * ys, xz = q.x * zs;
    const double yy = q.y * ys, yz = q.y * zs, zz = q.z * zs;
    return M33{{{1.0 - (yy + zz), xy - wz, xz + wy}, {xy + wz, 1.0 - (xx + zz), yz - wx}, {xz - wy, yz + wx, 1.0 - (xx + yy)}}};
  }
  double tdotx(const V3 &v) const { return r[0].x * v.x + r[1].x * v.y + r[2].x * v.z; }
  double tdoty(const V3 &v) const { return r[0].y * v.x + r[1].y * v.y + r[2].y * v.z; }
  double tdotz(const V3 &v) const { return r[0].z * v.x + r[1].z * v.y + r[2].z * v.z; }
  M33 transpose() const { return M33{{{r[0].x, r[1].x, r[2].x}, {r[0].y, r[1].y, r[2].y}, {r[0].z, r[1].z, r[2].z}}}; }
  M33 operator*(const M33 &m) const {
    return M33{{{m.tdotx(r[0]), m.tdoty(r[0]), m.tdotz(r[0])},
                {m.tdotx(r[1]), m.tdoty(r[1]), m.tdotz(r[1])},
                {m.tdotx(r[2]), m.tdoty(r[2]), m.tdotz(r[2])}}};
  }
  V3 operator*(const V3 &v) const { return V3{dot(r[0], v), dot(r[1], v), dot(r[2], v)}; }
  double at(int i, int j) const { return j == 0 ? r[i].x : (j == 1 ? r[i].y : r[i].z); }
  // Matrix3x3::getRotation
  Quat quaternion() const {
    const double trace = r[0].x + r[1].y + r[2].z;
    double t[4];
    if (trace > 0.0) {
      double s = std::sqrt(trace + 1.0);
      t[3] = s * 0.5;
      s = 0.5 / s;
      t[0] = (r[2].y - r[1].z) * s;
      t[1] = (r[0].z - r[2].x) * s;
      t[2] = (r[1].x - r[0].y) * s;
    } else {
      const int i = r[0].x < r[1].y ? (r[1].y < r[2].z ? 2 : 1) : (r[0].x < r[2].z ? 2 : 0);
      const int j = (i + 1) % 3, k = (i + 2) % 3;
      double s = std::sqrt(at(i, i) - at(j, j) - at(k, k) + 1.0);
      t[i] = s * 0.5;
      s = 0.5 / s;
      t[3] = (at(k, j) - at(j, k)) * s;
      t[j] = (at(j, i) + at(i, j)) * s;
      t[k] = (at(k, i) + at(i, k)) * s;
    }
    return Quat{t[0], t[1], t[2], t[3]};
  }
};

// Quaternion::setRPY (tf::createQuaternionFromRPY)
Quat quat_rpy(double roll, double pitch, double yaw) {
  const double hy = yaw * 0.5, hp = pitch * 0.5, hr = roll * 0.5;
  const double cy = std::cos(hy), sy = std::sin(hy), cp = std::cos(hp), sp = std::sin(hp), cr = std::cos(hr), sr = std::sin(hr);
  return Quat{sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy};
}

// tf::getYaw: Matrix3x3(q).getRPY(roll, pitch, yaw), solution 1 of getEulerYPR
double get_yaw(const Quat &q) {
  const M33 m = M33::rotation(q);
  if (std::fabs(m.r[2].x) >= 1) return 0.0;
  const double pitch = -std::asin(m.r[2].x);
  const double c = std::cos(pitch);
  return std::atan2(m.r[1].x / c, m.r[0].x / c);
}

struct Tf {
  M33 basis;
  V3 origin;
  static Tf identity() { return Tf{M33::identity(), V3{0, 0, 0}}; }
  static Tf from(const Quat &q, const V3 &t) { return Tf{M33::rotation(q), t}; }
  // Transform::operator()(x): x.dot3(basis rows) + origin
  V3 apply(const V3 &x) const {
    return V3{dot(x, basis.r[0]) + origin.x, dot(x, basis.r[1]) + origin.y, dot(x, basis.r[2]) + origin.z};
  }
  Tf operator*(const Tf &t) const { return Tf{basis * t.basis, apply(t.origin)}; }
  Tf inverse() const {
    const M33 inv = basis.transpose();
    return Tf{inv, inv * V3{-origin.x, -origin.y, -origin.z}};
  }
};

Tf tf_from_row(const double *r) { return Tf::from(Quat{r[3], r[4], r[5], r[6]}, V3{r[0], r[1], r[2]}); }

void tf_to_row(const Tf &t, double *out) {
  const Quat q = t.basis.quaternion();
  out[0] = t.origin.x; out[1] = t.origin.y; out[2] = t.origin.z;
  out[3] = q.x; out[4] = q.y; out[5] = q.z; out[6] = q.w;
}

// ---- roscpp Duration (roscpp_core rostime): fromSec and the (sec, nsec) comparison
struct Dur {
  int64_t sec, nsec;
  bool operator>(const Dur &o) const { return sec > o.sec || (sec == o.sec && nsec > o.nsec); }
};

// Time - Time: the two differences, normalised so that 0 <= nsec < 1e9 (normalizeSecNSecSigned)
Dur stamp_diff(uint32_t s1, uint32_t n1, uint32_t s0, uint32_t n0) {
  int64_t sec = (int64_t)(int32_t)s1 - (int64_t)(int32_t)s0, nsec = (int64_t)(int32_t)n1 - (int64_t)(int32_t)n0;
  int64_t nsec_part = nsec % 1000000000LL, sec_part = sec + nsec / 1000000000LL;
  if (nsec_part < 0) {
    nsec_part += 1000000000LL;
    --sec_part;
  }
  return Dur{(int64_t)(int32_t)sec_part, nsec_part};
}

}  // namespace

struct b2s_karto_node {
  b2s_karto_node_params prm{};
  b2s_laser laser{};
  int n_msg = 0, device = 0;
  bool inverted = false;
  Tf base_laser = Tf::identity();
  Dur interval{0, 0};
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
  const Tf base_laser = tf_from_row(laser_mount);
  const Tf laser_pose = base_laser * Tf::identity();
  const double offset[3] = {laser_pose.origin.x, laser_pose.origin.y, get_yaw(laser_pose.basis.quaternion())};
  const V3 up = base_laser.inverse().apply(V3{0, 0, 1 + laser_pose.origin.z});
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
  n->inverted = up.z <= 0;
  n->base_laser = base_laser;
  // ros::Duration::fromSec: sec = floor(d), nsec = round((d - sec) * 1e9), a rollover of nsec into sec
  int64_t sec = (int64_t)std::floor(iv), nsec = (int64_t)std::round((iv - (double)sec) * 1e9);
  sec += nsec / 1000000000LL;
  nsec %= 1000000000LL;
  n->interval = Dur{sec, nsec};
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
        const Tf odom_base = tf_from_row(row);
        const Tf op = odom_base * Tf::from(quat_rpy(0, 0, 0), V3{0, 0, 0});
        const double odom_pose[3] = {op.origin.x, op.origin.y, get_yaw(op.basis.quaternion())};
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
          const Tf corrected = Tf::from(quat_rpy(0, 0, pose[2]), V3{pose[0], pose[1], 0.0});
          const Tf odom_to_map = odom_base * corrected.inverse();
          const Tf mo = Tf::from(odom_to_map.basis.quaternion(), odom_to_map.origin).inverse();
          tf_to_row(mo, n->map_to_odom);
          const uint32_t *s = stamps + 2 * (size_t)i;
          if (!n->got_map || stamp_diff(s[0], s[1], n->last_map_sec, n->last_map_nsec) > n->interval) {
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
