// lesson5 motion de-skew as a device pre-stage (SURVEY.md §8(f).4): LidarUndistortion::CorrectLaserScan
// (lesson5/src/lidar_undistortion.cc:339-393) for a BATCH of LaserScans — every beam of every scan is one thread — with
// ComputeRotation (:396-430: linear interpolation in the integrated IMU angles) and ComputePosition (:433-445: linear
// in the odometry increment).  The per-scan preparation the node does under its queue locks is provided as host
// functions with the node's arithmetic: PruneImuDeque's angle integration (:196-238) and PruneOdomDeque's odometry
// increment (:296-333).  b2s_lidar_undistortion_node runs the whole node over a recording: the callbacks and both queue
// prunes on the host, then one CTA per published scan that integrates the scan's IMU queue into shared memory and
// corrects its beams.  b2s_deskew_node_* keeps B such nodes, one laser per recording, behind a handle that is fed in
// parts: the same host step per callback and the same kernel, over every recording's scans of a call in one launch.
//
// The beam angles are the node's angle cache (CreateAngleCache, :162-174), built on the host with its arithmetic: the
// angle in float from the LaserScan's float fields, its cos / sin from the C library in double.
//
// Pinned to the node (tests/test_deskew_reference.py, tests/test_gpu_deskew_edges.py) except for pcl::getTransformation
// and Eigen::Affine3f inverse and product: those are third-party header code that is not in the reference tree (PCL 1.8,
// Eigen 3.3), so their published algorithms are restated here (float arithmetic in Eigen's coefficient order, 3-term
// sums as a0 + (a1 + a2)), and the node's build uses stand-ins that restate them the same way.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "ros_math.cuh"

using namespace b2s;

namespace {

struct Affine3f {
  float m[3][3];
  float t[3];
};

__host__ __device__ inline float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); }  // Eigen's unrolled 3-term redux

// pcl::getTransformation (PCL common/impl/eigen.hpp): cos / sin are the C library's double functions, rounded to float
__host__ __device__ inline Affine3f get_transformation(float x, float y, float z, float roll, float pitch, float yaw) {
  const float A = (float)cos((double)yaw), B = (float)sin((double)yaw), C = (float)cos((double)pitch), D = (float)sin((double)pitch),
              E = (float)cos((double)roll), F = (float)sin((double)roll), DE = D * E, DF = D * F;
  Affine3f t;
  t.m[0][0] = A * C; t.m[0][1] = A * DF - B * E; t.m[0][2] = B * F + A * DE; t.t[0] = x;
  t.m[1][0] = B * C; t.m[1][1] = A * E + B * DF; t.m[1][2] = B * DE - A * F; t.t[1] = y;
  t.m[2][0] = -D;    t.m[2][1] = C * F;          t.m[2][2] = C * E;          t.t[2] = z;
  return t;
}

__host__ __device__ inline float cofactor(const float m[3][3], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
}

// Transform<float, 3, Affine>::inverse(): cofactor inverse of the linear part (compute_inverse_size3), t' = -(L^-1 t)
__host__ __device__ inline Affine3f affine_inverse(const Affine3f &a) {
  Affine3f r;
  const float c0 = cofactor(a.m, 0, 0), c1 = cofactor(a.m, 1, 0), c2 = cofactor(a.m, 2, 0);
  const float det = sum3(c0 * a.m[0][0], c1 * a.m[1][0], c2 * a.m[2][0]);
  const float invdet = 1.0f / det;
  r.m[0][0] = c0 * invdet; r.m[0][1] = c1 * invdet; r.m[0][2] = c2 * invdet;
  r.m[1][0] = cofactor(a.m, 0, 1) * invdet; r.m[1][1] = cofactor(a.m, 1, 1) * invdet; r.m[1][2] = cofactor(a.m, 2, 1) * invdet;
  r.m[2][0] = cofactor(a.m, 0, 2) * invdet; r.m[2][1] = cofactor(a.m, 1, 2) * invdet; r.m[2][2] = cofactor(a.m, 2, 2) * invdet;
#pragma unroll
  for (int i = 0; i < 3; i++) r.t[i] = -sum3(r.m[i][0] * a.t[0], r.m[i][1] * a.t[1], r.m[i][2] * a.t[2]);
  return r;
}

// Affine * Affine: linear = L1 L2, translation = L1 t2 + t1
__host__ __device__ inline Affine3f affine_mul(const Affine3f &a, const Affine3f &b) {
  Affine3f r;
#pragma unroll
  for (int i = 0; i < 3; i++) {
#pragma unroll
    for (int j = 0; j < 3; j++) r.m[i][j] = sum3(a.m[i][0] * b.m[0][j], a.m[i][1] * b.m[1][j], a.m[i][2] * b.m[2][j]);
    r.t[i] = sum3(a.m[i][0] * b.t[0], a.m[i][1] * b.t[1], a.m[i][2] * b.t[2]) + a.t[i];
  }
  return r;
}

__host__ __device__ inline bool reading_valid(float r, const b2s_deskew_scan &s) {
  return isfinite(r) && !(r < s.range_min) && !(r > s.range_max);  // (:349-352)
}

// the pose of the sensor at the time of beam i, relative to the odometry / IMU origin of the scan
__device__ inline Affine3f pose_at(const b2s_deskew_scan &s, const double *__restrict__ imu_time, const double *__restrict__ rx,
                                   const double *__restrict__ ry, const double *__restrict__ rz, int i) {
  const double t = s.time_start + i * s.time_increment;
  float rotx = 0, roty = 0, rotz = 0, posx = 0, posy = 0, posz = 0;
  if (s.use_imu) {  // ComputeRotation
    int front = 0;
    while (front < s.imu_last) {
      if (t < imu_time[front]) break;
      ++front;
    }
    if (t > imu_time[front] || front == 0) {
      rotx = (float)rx[front]; roty = (float)ry[front]; rotz = (float)rz[front];
    } else {
      const int back = front - 1;
      const double rf = (t - imu_time[back]) / (imu_time[front] - imu_time[back]);
      const double rb = (imu_time[front] - t) / (imu_time[front] - imu_time[back]);
      rotx = (float)(rx[front] * rf + rx[back] * rb);
      roty = (float)(ry[front] * rf + ry[back] * rb);
      rotz = (float)(rz[front] * rf + rz[back] * rb);
    }
  }
  if (s.use_odom) {  // ComputePosition
    const double ratio = (t - s.odom_start_time) / (s.odom_end_time - s.odom_start_time);
    posx = (float)(s.odom_incre[0] * ratio); posy = (float)(s.odom_incre[1] * ratio); posz = (float)(s.odom_incre[2] * ratio);
  }
  return get_transformation(posx, posy, posz, rotx, roty, rotz);
}

// CorrectLaserScan's body for one valid reading (:358-393): beam i of range `range` at (cos, sin) = cs, moved by the
// inverted pose of the scan's first valid reading
__device__ inline void deskew_beam(const b2s_deskew_scan &s, const Affine3f &inv, const double *__restrict__ it,
                                   const double *__restrict__ rx, const double *__restrict__ ry, const double *__restrict__ rz,
                                   int i, float range, double2 cs, float *__restrict__ o) {
  const double px = range * cs.x, py = range * cs.y, pz = 1.0;
  const Affine3f bt = affine_mul(inv, pose_at(s, it, rx, ry, rz, i));
  o[0] = (float)(bt.m[0][0] * px + bt.m[0][1] * py + bt.m[0][2] * pz + bt.t[0]);
  o[1] = (float)(bt.m[1][0] * px + bt.m[1][1] * py + bt.m[1][2] * pz + bt.t[1]);
  o[2] = (float)(bt.m[2][0] * px + bt.m[2][1] * py + bt.m[2][2] * pz + bt.t[2]);
}

// PruneImuDeque's integration loop (:207-246) over the n messages of the pruned queue: stamp[i], angular velocity
// (wx, wy, wz)[i * wstride].  Returns current_imu_index_ after the loop's final decrement, or -2 where the node reads
// imu_time_[-1] (a message at or after the scan start before any message before it) or writes entry `cap` of its table.
// STORE fills the table (entry 0 is left alone when no message precedes the scan); without it the entries are only
// counted.
constexpr int IMU_QUEUE_LENGTH = 2000;  // queueLength (:20)

template <bool STORE>
__host__ __device__ inline int imu_table(int n, const double *stamp, const double *wx, const double *wy, const double *wz,
                                         int wstride, double scan_start, double scan_end, int cap, double *imu_time,
                                         double *rot_x, double *rot_y, double *rot_z) {
  int idx = 0;
  for (int i = 0; i < n; i++) {
    const double t = stamp[i];
    if (t < scan_start) {
      if (idx == 0) {
        if (STORE) {
          rot_x[0] = rot_y[0] = rot_z[0] = 0.0;
          imu_time[0] = t;
        }
        ++idx;
      }
      continue;
    }
    if (t > scan_end) break;
    if (idx == 0 || idx >= cap) return -2;
    if (STORE) {
      const double dt = t - imu_time[idx - 1];
      rot_x[idx] = rot_x[idx - 1] + wx[(size_t)i * wstride] * dt;
      rot_y[idx] = rot_y[idx - 1] + wy[(size_t)i * wstride] * dt;
      rot_z[idx] = rot_z[idx - 1] + wz[(size_t)i * wstride] * dt;
      imu_time[idx] = t;
    }
    ++idx;
  }
  return idx - 1;
}

// One CTA per (scan, slab of beams): scans on x, whose limit is 2^31 - 1, so a whole recording is one launch; slabs on y.
// The reference takes transStartInverse from the FIRST VALID reading of the scan (first_point_flag): every CTA finds
// that beam with a block-wide minimum, thread 0 inverts its pose once.
constexpr int DSK_THREADS = 256;
__global__ void __launch_bounds__(DSK_THREADS)
    k_deskew(const float *__restrict__ ranges, int n_beams, const double2 *__restrict__ angle_cs,
             const b2s_deskew_scan *__restrict__ scans, const double *__restrict__ imu_time, const double *__restrict__ imu_rx,
             const double *__restrict__ imu_ry, const double *__restrict__ imu_rz, int imu_stride, float *__restrict__ out_xyz) {
  const int b = blockIdx.x;
  const b2s_deskew_scan s = scans[b];
  const float *r = ranges + (size_t)b * n_beams;
  const double *it = imu_time + (size_t)b * imu_stride, *rx = imu_rx + (size_t)b * imu_stride,
               *ry = imu_ry + (size_t)b * imu_stride, *rz = imu_rz + (size_t)b * imu_stride;
  __shared__ int s_first;
  __shared__ Affine3f s_inv;
  if (threadIdx.x == 0) s_first = n_beams;
  __syncthreads();
  int mine = n_beams;
  for (int i = threadIdx.x; i < n_beams; i += DSK_THREADS)
    if (reading_valid(r[i], s)) { mine = i; break; }
  if (mine < n_beams) atomicMin(&s_first, mine);
  __syncthreads();
  if (threadIdx.x == 0 && s_first < n_beams) s_inv = affine_inverse(pose_at(s, it, rx, ry, rz, s_first));
  __syncthreads();
  const int i = blockIdx.y * DSK_THREADS + threadIdx.x;
  if (i >= n_beams) return;
  float *o = out_xyz + ((size_t)b * n_beams + i) * 3;
  const float range = r[i];
  if (!reading_valid(range, s)) {  // the cloud is cleared and resized per scan (:62, :139): skipped points stay default
    o[0] = o[1] = o[2] = 0.0f;
    return;
  }
  deskew_beam(s, s_inv, it, rx, ry, rz, i, range, angle_cs[i] /* a_cos_[i], a_sin_[i] */, o);
}

// ---- the node over recordings (b2s_deskew_node_*, and b2s_lidar_undistortion_node as a batch of one) ----

// a published scan of any recording in the call: where its ranges are (the call's upload, or the held-scan store for
// the scan a call's first callback corrects), its cloud's first beam in the call's output, its recording's angle cache,
// the pruned IMU queue as [imu_lo, imu_lo + imu_n) of the call's packed log, and its scan end
struct NodeRow {
  long long ranges, out, angles, imu_lo;
  int32_t n_beams, imu_n, held, reserved;
  double scan_end;
};

// after the node kernel: a recording's last scan of the call, [src, src + n) of the upload, becomes its held scan at dst
struct HoldCopy {
  long long src, dst;
  int32_t n, reserved;
};

// One CTA per published scan of every recording in the call (grid x, up to 2^31 - 1 scans).  Thread 0 integrates the
// scan's IMU queue from the log into shared memory, [4][stride] doubles with stride the call's largest table; entry 0
// is zeroed first, so that imu_last = -1 (no message before the scan start) takes rotation 0 as the node's reset table
// gives.  Then the CTA finds the first valid reading, thread 0 inverts its pose once, and the CTA walks all beams.
constexpr int NODE_THREADS = 256;
__global__ void __launch_bounds__(NODE_THREADS)
    k_deskew_node(const float *__restrict__ ranges, const float *__restrict__ held, const double2 *__restrict__ angle_cs,
                  const NodeRow *__restrict__ rows, const b2s_deskew_scan *__restrict__ states,
                  const double *__restrict__ log_t, const double *__restrict__ log_x, const double *__restrict__ log_y,
                  const double *__restrict__ log_z, int stride, float *__restrict__ out_xyz) {
  extern __shared__ double s_tab[];
  double *it = s_tab, *rx = s_tab + stride, *ry = rx + stride, *rz = ry + stride;
  const NodeRow w = rows[blockIdx.x];
  const b2s_deskew_scan s = states[blockIdx.x];
  const int n_beams = w.n_beams;
  const float *r = (w.held ? held : ranges) + w.ranges;
  const double2 *cs = angle_cs + w.angles;
  float *out = out_xyz + w.out * 3;
  __shared__ int s_first;
  __shared__ Affine3f s_inv;
  if (threadIdx.x == 0) {
    s_first = n_beams;
    if (s.use_imu) {
      it[0] = rx[0] = ry[0] = rz[0] = 0.0;
      imu_table<true>(w.imu_n, log_t + w.imu_lo, log_x + w.imu_lo, log_y + w.imu_lo, log_z + w.imu_lo, 1, s.time_start,
                      w.scan_end, IMU_QUEUE_LENGTH, it, rx, ry, rz);
    }
  }
  __syncthreads();
  int mine = n_beams;
  for (int i = threadIdx.x; i < n_beams; i += NODE_THREADS)
    if (reading_valid(r[i], s)) { mine = i; break; }
  if (mine < n_beams) atomicMin(&s_first, mine);
  __syncthreads();
  if (threadIdx.x == 0 && s_first < n_beams) s_inv = affine_inverse(pose_at(s, it, rx, ry, rz, s_first));
  __syncthreads();
  for (int i = threadIdx.x; i < n_beams; i += NODE_THREADS) {
    float *o = out + (size_t)i * 3;
    const float range = r[i];
    if (!reading_valid(range, s)) {
      o[0] = o[1] = o[2] = 0.0f;
      continue;
    }
    deskew_beam(s, s_inv, it, rx, ry, rz, i, range, cs[i], o);
  }
}

// one CTA per recording with a scan in the call: its last scan becomes the held scan.  Enqueued after k_deskew_node,
// which may still read the previous held scan from the same store.
__global__ void k_deskew_node_hold(const float *__restrict__ ranges, const HoldCopy *__restrict__ copies, float *held) {
  const HoldCopy c = copies[blockIdx.x];
  for (int i = threadIdx.x; i < c.n; i += blockDim.x) held[c.dst + i] = ranges[c.src + i];
}

// (x, y, z, roll, pitch, yaw) of an odometry message as PruneOdomDeque takes it (:304-325): tf::quaternionMsgToTF, then
// tf::Matrix3x3(q).getRPY
void odom_pose(const b2s_odom_msg &m, double out[6]) {
  TfTransform t;
  tf_set_rotation(t, m.orientation);
  out[0] = m.position[0];
  out[1] = m.position[1];
  out[2] = m.position[2];
  tf_get_rpy(t, out[3], out[4], out[5]);
}

// What one LidarUndistortion node keeps from one callback to the next.
struct NodeState {
  bool seen = false;               // the first-scan flag: the node has cached a scan (:136)
  b2s_deskew_node_scan held{};     // the scan in the laser queue: stamp and float fields (its ranges: the held store)
  std::vector<b2s_imu_msg> imu;    // the IMU deque: messages not yet pruned, in delivery order
  std::vector<b2s_odom_msg> odom;  // the odometry deque
  b2s_odom_msg start_msg{}, end_msg{};  // start_odom_msg_ / end_odom_msg_: all zero bytes is the default-constructed
                                        // message (stamp 0, zero quaternion)
};

// A call's view of one recording's queues: the deque kept from earlier calls followed by the call's new messages.  The
// queues are [ilo, imu_hi) and [olo, odom_hi) of these logs; the prunes advance ilo and olo.
struct NodeLogs {
  const double *imu_t;         // stamps of the IMU log (the first column of the call's packed log)
  const b2s_odom_msg *odom;    // the odometry log
  const double *odom_t;        // its stamps
  int ilo, olo;
};

// One callback's correction of the held scan R.held, with the IMU and odometry queues reaching imu_hi / odom_hi of the
// logs (CacheLaserScan pops it, :145-150; PruneImuDeque, :177-249; PruneOdomDeque, :252-336).  Returns the row's
// status and fills its state s and, for a published row, w.imu_lo (relative to the recording's log), w.imu_n and
// w.scan_end.
int32_t correct_held(const b2s_deskew_laser &L, NodeState &R, NodeLogs &g, int imu_hi, int odom_hi, b2s_deskew_scan &s,
                     NodeRow &w) {
  const double scan_count = (double)L.n_beams;  // scan_count_, a double member, from the first scan (:136)
  const b2s_deskew_node_scan &sc = R.held;
  const double start = ros_time_to_sec(sc.sec, sc.nsec), inc = sc.time_increment, end = start + inc * (scan_count - 1);
  int32_t status = B2S_DESKEW_PUBLISHED;
  std::memset(&s, 0, sizeof s);
  w.scan_end = end;
  s.time_start = start;
  s.time_increment = inc;
  s.range_min = sc.range_min;
  s.range_max = sc.range_max;
  s.use_imu = L.use_imu != 0;
  s.use_odom = L.use_odom != 0;
  if (L.use_imu) {  // PruneImuDeque (:177-249)
    const double *t = g.imu_t;
    if (g.ilo == imu_hi || t[g.ilo] > start || t[imu_hi - 1] < end) return B2S_DESKEW_WAIT_IMU;
    while (g.ilo < imu_hi && t[g.ilo] < start - 0.1) ++g.ilo;
    if (g.ilo == imu_hi) return B2S_DESKEW_IMU_EMPTY;
    w.imu_lo = g.ilo;
    w.imu_n = imu_hi - g.ilo;
    s.imu_last = imu_table<false>(w.imu_n, t + g.ilo, nullptr, nullptr, nullptr, 0, start, end, IMU_QUEUE_LENGTH, nullptr,
                                  nullptr, nullptr, nullptr);
    if (s.imu_last == -2) status = B2S_DESKEW_UNDEFINED;  // the odometry queue is still pruned, as the node goes on
  }
  if (L.use_odom) {  // PruneOdomDeque (:252-336)
    const double *t = g.odom_t;
    if (g.olo == odom_hi || t[g.olo] > start || t[odom_hi - 1] < end)
      return status == B2S_DESKEW_PUBLISHED ? B2S_DESKEW_WAIT_ODOM : status;
    while (g.olo < odom_hi && t[g.olo] < start - 0.1) ++g.olo;
    if (g.olo == odom_hi) return status == B2S_DESKEW_PUBLISHED ? B2S_DESKEW_ODOM_EMPTY : status;
    for (int i = g.olo; i < odom_hi; i++) {
      if (t[i] < start) {
        R.start_msg = g.odom[i];
        continue;
      }
      if (t[i] <= end)
        R.end_msg = g.odom[i];
      else
        break;
    }
    double sp[6], ep[6];
    odom_pose(R.start_msg, sp);
    odom_pose(R.end_msg, ep);
    s.odom_start_time = ros_time_to_sec(R.start_msg.sec, R.start_msg.nsec);
    s.odom_end_time = ros_time_to_sec(R.end_msg.sec, R.end_msg.nsec);
    b2s_deskew_odom_increment(sp, ep, s.odom_incre);
  }
  return status;
}

}  // namespace

// B LidarUndistortion nodes, one laser per recording.  b2s_lidar_undistortion_node builds one of batch 1 per call.
struct b2s_deskew_node {
  Stream st;  // declared first: destroyed after the buffers
  int device = 0, batch = 0;
  bool failed = false;  // a device error: the nodes' state is lost
  std::vector<b2s_deskew_laser> lasers;
  std::vector<long long> beam_off;  // recording b's first beam in the angle cache and the held store
  std::vector<NodeState> rec;
  const double2 *angle_cs = nullptr;  // [sum n_beams]: CreateAngleCache (:162-174) of every recording, on the device
  Buf<double2> angles;                // the handle's angle_cs (a one-shot call's is stream-ordered memory of the call)
  Buf<float> held;                    // [sum n_beams]: every recording's held scan (unallocated for a one-shot call)
};

namespace {

// the nodes' host state, and their angle caches on the host (cs) for the caller to upload
void nodes_init(b2s_deskew_node &h, int batch, const b2s_deskew_laser *lasers, int device, std::vector<double2> &cs) {
  h.device = device;
  h.batch = batch;
  h.lasers.assign(lasers, lasers + batch);
  h.rec.assign(batch, NodeState());
  h.beam_off.resize(batch + 1);
  h.beam_off[0] = 0;
  for (int b = 0; b < batch; b++) h.beam_off[b + 1] = h.beam_off[b] + lasers[b].n_beams;
  const size_t nb = (size_t)h.beam_off[batch];
  // CreateAngleCache: angle_min and angle_increment are float fields of the LaserScan and i is unsigned, so the angle is
  // summed in float and only widened for the double cos / sin
  cs.resize(nb);
  for (int b = 0; b < batch; b++)
    for (int i = 0; i < lasers[b].n_beams; i++) {
      const float step = (float)(unsigned)i * lasers[b].angle_increment;
      const double angle = lasers[b].angle_min + step;
      cs[h.beam_off[b] + i] = make_double2(cos(angle), sin(angle));
    }
}

// The refusals of b2s_deskew_node_process, before anything is written: counts and arrays, and arrival counts that
// decrease or exceed their log.  imu_first / odom_first [B + 1] get every recording's first message of the call.
b2s_status nodes_check(const b2s_deskew_node &h, const int32_t *n_scans, const b2s_deskew_node_scan *scans,
                       const float *ranges, const int32_t *n_imu, const b2s_imu_msg *imu, const int32_t *n_odom,
                       const b2s_odom_msg *odom, const int32_t *out_status, const float *out_xyz,
                       std::vector<long long> &scan_first, std::vector<long long> &imu_first,
                       std::vector<long long> &odom_first) {
  const int B = h.batch;
  if (!n_scans || !n_imu || !n_odom)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_process: null count array");
  scan_first.assign(B + 1, 0);
  imu_first.assign(B + 1, 0);
  odom_first.assign(B + 1, 0);
  bool any_imu_flag = false, any_odom_flag = false;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0 || n_imu[b] < 0 || n_odom[b] < 0)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_process: negative count");
    scan_first[b + 1] = scan_first[b] + n_scans[b];
    imu_first[b + 1] = imu_first[b] + n_imu[b];
    odom_first[b + 1] = odom_first[b] + n_odom[b];
    any_imu_flag |= h.lasers[b].use_imu != 0;
    any_odom_flag |= h.lasers[b].use_odom != 0;
  }
  if ((scan_first[B] > 0 && (!scans || !ranges || !out_status || !out_xyz)) || (imu_first[B] > 0 && !imu) ||
      (odom_first[B] > 0 && !odom) || (any_imu_flag && !imu) || (any_odom_flag && !odom))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_process: null array where a count is non-zero or a flag is on");
  if (scan_first[B] > 0x7fffffffLL)
    B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_deskew_node_process: more than 2^31 - 1 scans in one call");
  for (int b = 0; b < B; b++)
    for (long long k = scan_first[b]; k < scan_first[b + 1]; k++) {
      const int ip = k > scan_first[b] ? scans[k - 1].imu_arrived : 0, op = k > scan_first[b] ? scans[k - 1].odom_arrived : 0;
      if (scans[k].imu_arrived < ip || scans[k].imu_arrived > n_imu[b] || scans[k].odom_arrived < op ||
          scans[k].odom_arrived > n_odom[b])
        B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_process: arrival counts decrease or exceed their log");
    }
  return B2S_OK;
}

// The callbacks of one call for every recording, on the host, then one node kernel over every published row.  Inputs
// are checked (nodes_check).  Callback k of recording b writes output row scan_first[b] + k - shift: shift 0 is the
// handle's callback-indexed rows; shift 1 the one-shot call's rows indexed by the corrected scan, whose caching first
// callback writes no row and whose last row (the held scan) the caller writes.  out_state may be NULL.
b2s_status nodes_process(b2s_deskew_node &h, int shift, const int32_t *n_scans, const b2s_deskew_node_scan *scans,
                         const float *ranges, const b2s_imu_msg *imu, const b2s_odom_msg *odom,
                         const std::vector<long long> &scan_first, const std::vector<long long> &imu_first,
                         const std::vector<long long> &odom_first, int32_t *out_status, b2s_deskew_scan *out_state,
                         float *out_xyz) {
  const int B = h.batch;
  // ---- every recording's IMU log of the call, as SoA doubles (t, x, y, z): its kept deque, then the new messages
  std::vector<long long> log_off(B + 1, 0), range_off(B + 1, 0);  // range_off: also each recording's first output beam
  for (int b = 0; b < B; b++) {
    const long long n_log = h.lasers[b].use_imu ? (long long)h.rec[b].imu.size() + (imu_first[b + 1] - imu_first[b]) : 0;
    log_off[b + 1] = log_off[b] + n_log;
    range_off[b + 1] = range_off[b] + (long long)n_scans[b] * h.lasers[b].n_beams;
  }
  const size_t n_log = (size_t)log_off[B], nr = (size_t)range_off[B];
  std::vector<double> pack(4 * n_log);
  for (int b = 0; b < B; b++) {
    if (!h.lasers[b].use_imu) continue;
    const std::vector<b2s_imu_msg> &kept = h.rec[b].imu;
    for (long long i = log_off[b]; i < log_off[b + 1]; i++) {
      const long long j = i - log_off[b];
      const b2s_imu_msg &m = j < (long long)kept.size() ? kept[j] : imu[imu_first[b] + j - (long long)kept.size()];
      pack[i] = ros_time_to_sec(m.sec, m.nsec);
      for (int a = 0; a < 3; a++) pack[(a + 1) * n_log + i] = m.angular_velocity[a];
    }
  }

  // ---- the callbacks
  std::vector<NodeRow> rows;
  std::vector<b2s_deskew_scan> states;
  std::vector<HoldCopy> holds;
  std::vector<b2s_odom_msg> olog;
  std::vector<double> olog_t;
  int stride = 1;  // the largest IMU table of a published scan
  for (int b = 0; b < B; b++) {
    const b2s_deskew_laser &L = h.lasers[b];
    NodeState &R = h.rec[b];
    const int n_new_imu = L.use_imu ? (int)(imu_first[b + 1] - imu_first[b]) : 0;
    const int n_new_odom = L.use_odom ? (int)(odom_first[b + 1] - odom_first[b]) : 0;
    const int kept_imu = (int)R.imu.size(), kept_odom = (int)R.odom.size();
    olog.assign(R.odom.begin(), R.odom.end());
    if (n_new_odom) olog.insert(olog.end(), odom + odom_first[b], odom + odom_first[b] + n_new_odom);
    olog_t.resize(olog.size());
    for (size_t i = 0; i < olog.size(); i++) olog_t[i] = ros_time_to_sec(olog[i].sec, olog[i].nsec);
    NodeLogs g = {pack.data() + log_off[b], olog.data(), olog_t.data(), 0, 0};
    for (int k = 0; k < n_scans[b]; k++) {
      const long long q = scan_first[b] + k, row = q - shift;
      const b2s_deskew_node_scan &sc = scans[q];
      b2s_deskew_scan s;
      std::memset(&s, 0, sizeof s);
      int32_t status = B2S_DESKEW_CACHED;
      NodeRow w = {};
      if (R.seen) {
        status = correct_held(L, R, g, kept_imu + (L.use_imu ? sc.imu_arrived : 0), kept_odom + (L.use_odom ? sc.odom_arrived : 0),
                              s, w);
      }
      R.seen = true;
      R.held = sc;
      if (row < 0) continue;
      out_status[row] = status;
      const bool keep = status == B2S_DESKEW_PUBLISHED || status == B2S_DESKEW_UNDEFINED;
      if (out_state) {
        if (keep)
          out_state[row] = s;
        else
          std::memset(&out_state[row], 0, sizeof s);
      }
      if (status == B2S_DESKEW_PUBLISHED) {
        w.held = k == 0;
        w.ranges = k == 0 ? h.beam_off[b] : range_off[b] + (long long)(k - 1) * L.n_beams;
        w.out = range_off[b] + (long long)(k - shift) * L.n_beams;
        w.angles = h.beam_off[b];
        w.imu_lo += log_off[b];
        w.n_beams = L.n_beams;
        rows.push_back(w);
        states.push_back(s);
        if (L.use_imu) stride = std::max(stride, s.imu_last + 1);
      }
    }
    // the deques after the call: what the prunes left, and every message of the call (those after the last scan are
    // delivered before the next call's first scan)
    if (L.use_imu) {
      std::vector<b2s_imu_msg> next;
      next.reserve(kept_imu + n_new_imu - g.ilo);
      for (int j = g.ilo; j < kept_imu + n_new_imu; j++) next.push_back(j < kept_imu ? R.imu[j] : imu[imu_first[b] + j - kept_imu]);
      R.imu.swap(next);
    }
    if (L.use_odom) R.odom.assign(olog.begin() + g.olo, olog.end());
    if (n_scans[b] > 0 && h.held.p)
      holds.push_back(HoldCopy{range_off[b] + (long long)(n_scans[b] - 1) * L.n_beams, h.beam_off[b], L.n_beams, 0});
  }
  const size_t n_pub = rows.size(), n_out = nr;
  if (n_pub == 0 && n_out) std::memset(out_xyz, 0, n_out * 3 * sizeof(float));
  if (n_pub == 0 && holds.empty()) return B2S_OK;

  // ---- one upload of the call's small inputs after the ranges: the IMU logs, the published rows' states and rows, and
  // the held-scan copies
  const size_t off_states = 4 * n_log, off_rows = off_states + n_pub * sizeof(b2s_deskew_scan) / sizeof(double);
  const size_t off_holds = off_rows + n_pub * sizeof(NodeRow) / sizeof(double);
  static_assert(sizeof(b2s_deskew_scan) % sizeof(double) == 0 && sizeof(NodeRow) % sizeof(double) == 0 &&
                    sizeof(HoldCopy) % sizeof(double) == 0, "packing");
  pack.resize(off_holds + holds.size() * sizeof(HoldCopy) / sizeof(double));
  std::memcpy(pack.data() + off_states, states.data(), n_pub * sizeof(b2s_deskew_scan));
  std::memcpy(pack.data() + off_rows, rows.data(), n_pub * sizeof(NodeRow));
  std::memcpy(pack.data() + off_holds, holds.data(), holds.size() * sizeof(HoldCopy));

  cudaStream_t st = h.st;
  const size_t smem = 4 * sizeof(double) * (size_t)stride;  // at most 2000 entries: 64 000 bytes
  if (smem > 48 * 1024) B2S_CUDA_CHECK(raise_dyn_smem(k_deskew_node, smem));
  AsyncBuf<float> d_r(st), d_o(st);
  AsyncBuf<double> d_pack(st);
  B2S_CUDA_CHECK(d_r.alloc(nr));
  B2S_CUDA_CHECK(d_pack.alloc(pack.size()));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, nr * sizeof(float), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_pack, pack.data(), pack.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  if (n_pub) {
    B2S_CUDA_CHECK(d_o.alloc(n_out * 3));
    // rows the kernel does not write are zero bytes: one memset per run of unpublished rows
    for (size_t p = 0, next = 0; p <= n_pub; p++) {
      const size_t until = p < n_pub ? (size_t)rows[p].out : n_out;
      if (until > next) B2S_CUDA_CHECK(cudaMemsetAsync(d_o + next * 3, 0, (until - next) * 3 * sizeof(float), st));
      if (p < n_pub) next = until + rows[p].n_beams;
    }
    const double *log = d_pack;
    k_deskew_node<<<(unsigned)n_pub, NODE_THREADS, smem, st>>>(
        d_r, h.held, h.angle_cs, reinterpret_cast<const NodeRow *>(d_pack + off_rows),
        reinterpret_cast<const b2s_deskew_scan *>(d_pack + off_states), log, log + n_log, log + 2 * n_log, log + 3 * n_log,
        stride, d_o);
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  if (!holds.empty()) {
    k_deskew_node_hold<<<(unsigned)holds.size(), NODE_THREADS, 0, st>>>(
        d_r, reinterpret_cast<const HoldCopy *>(d_pack + off_holds), h.held);
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  if (n_pub) B2S_CUDA_CHECK(cudaMemcpyAsync(out_xyz, d_o, n_out * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  return B2S_OK;
}

}  // namespace

extern "C" {

int32_t b2s_deskew_integrate_imu(int n_imu, const double *stamp, const double *angular_velocity, double scan_time_start,
                                 double scan_time_end, int capacity, double *imu_time, double *rot_x, double *rot_y,
                                 double *rot_z) {
  if (n_imu < 0 || capacity < 1 || !imu_time || !rot_x || !rot_y || !rot_z || (n_imu > 0 && (!stamp || !angular_velocity))) return -2;
  for (int i = 0; i < capacity; i++) imu_time[i] = rot_x[i] = rot_y[i] = rot_z[i] = 0.0;  // ResetParameters (:66-74)
  return imu_table<true>(n_imu, stamp, angular_velocity, angular_velocity + 1, angular_velocity + 2, 3, scan_time_start,
                         scan_time_end, capacity, imu_time, rot_x, rot_y, rot_z);
}

void b2s_deskew_odom_increment(const double start_pose[6], const double end_pose[6], float out_increment[3]) {
  if (!start_pose || !end_pose || !out_increment) return;
  const Affine3f b = get_transformation((float)start_pose[0], (float)start_pose[1], (float)start_pose[2], (float)start_pose[3],
                                        (float)start_pose[4], (float)start_pose[5]);
  const Affine3f e = get_transformation((float)end_pose[0], (float)end_pose[1], (float)end_pose[2], (float)end_pose[3],
                                        (float)end_pose[4], (float)end_pose[5]);
  const Affine3f bt = affine_mul(affine_inverse(b), e);
  out_increment[0] = bt.t[0]; out_increment[1] = bt.t[1]; out_increment[2] = bt.t[2];
}

b2s_status b2s_lidar_undistort(int batch, int n_beams, const float *ranges, double angle_min, double angle_increment,
                               const b2s_deskew_scan *scans, const double *imu_time, const double *imu_rot_x,
                               const double *imu_rot_y, const double *imu_rot_z, int imu_stride, float *out_xyz, int device,
                               void *cuda_stream) {
  B2S_NVTX("LidarUndistortion::CorrectLaserScan (batch)");
  if (batch < 0 || n_beams < 1 || imu_stride < 1 || !ranges || !scans || !imu_time || !imu_rot_x || !imu_rot_y || !imu_rot_z || !out_xyz)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistort: null argument or empty scan");
  if (batch == 0) return B2S_OK;
  if (ceil_div(n_beams, DSK_THREADS) > 65535) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistort: more than 65535 * 256 beams");
  for (int b = 0; b < batch; b++) {
    if (scans[b].imu_last < 0 || scans[b].imu_last >= imu_stride)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistort: imu_last outside the IMU table");
    if (scans[b].use_odom && !(scans[b].odom_end_time != scans[b].odom_start_time))
      B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistort: odometry interval of zero length");
  }
  // CreateAngleCache (:162-174): angle_min and angle_increment are float fields of the LaserScan and i is unsigned, so
  // the angle is summed in float and only widened for the double cos / sin
  const float amin = (float)angle_min, ainc = (float)angle_increment;
  std::vector<double> angle_cs(2 * (size_t)n_beams);
  for (int i = 0; i < n_beams; i++) {
    const float step = (float)(unsigned)i * ainc;
    const double angle = amin + step;
    angle_cs[2 * i] = cos(angle);
    angle_cs[2 * i + 1] = sin(angle);
  }
  if (b2s_status st = open_device(device)) return st;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  const size_t nr = (size_t)batch * n_beams, ni = (size_t)batch * imu_stride;
  AsyncBuf<float> d_r(st), d_o(st);
  AsyncBuf<double> d_imu(st), d_ang(st);
  AsyncBuf<b2s_deskew_scan> d_s(st);
  B2S_CUDA_CHECK(d_r.alloc(nr));
  B2S_CUDA_CHECK(d_o.alloc(nr * 3));
  B2S_CUDA_CHECK(d_imu.alloc(ni * 4));
  B2S_CUDA_CHECK(d_ang.alloc(angle_cs.size()));
  B2S_CUDA_CHECK(d_s.alloc(batch));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, nr * sizeof(float), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_ang, angle_cs.data(), angle_cs.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_imu, imu_time, ni * sizeof(double), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_imu + ni, imu_rot_x, ni * sizeof(double), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_imu + 2 * ni, imu_rot_y, ni * sizeof(double), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_imu + 3 * ni, imu_rot_z, ni * sizeof(double), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_s, scans, (size_t)batch * sizeof(b2s_deskew_scan), cudaMemcpyHostToDevice, st));
  const dim3 grid(batch, ceil_div(n_beams, DSK_THREADS));
  k_deskew<<<grid, DSK_THREADS, 0, st>>>(d_r, n_beams, reinterpret_cast<const double2 *>(static_cast<double *>(d_ang)), d_s,
                                         d_imu, d_imu + ni, d_imu + 2 * ni, d_imu + 3 * ni, imu_stride, d_o);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out_xyz, d_o, nr * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  return B2S_OK;
}

b2s_status b2s_lidar_undistortion_node(int use_imu, int use_odom, float angle_min, float angle_increment, int n_beams,
                                       int n_scans, const b2s_deskew_node_scan *scans, const float *ranges, int n_imu,
                                       const b2s_imu_msg *imu, int n_odom, const b2s_odom_msg *odom, int32_t *out_status,
                                       b2s_deskew_scan *out_state, float *out_xyz, int device, void *cuda_stream) {
  B2S_NVTX("LidarUndistortion node (recording)");
  if (n_scans < 0 || n_imu < 0 || n_odom < 0 || n_beams < 1 || !scans || !ranges || !out_status || !out_xyz ||
      (use_imu && !imu) || (use_odom && !odom))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistortion_node: null argument, negative count or empty scan");
  for (int k = 0; k < n_scans; k++) {
    const int ip = k ? scans[k - 1].imu_arrived : 0, op = k ? scans[k - 1].odom_arrived : 0;
    if (scans[k].imu_arrived < ip || scans[k].imu_arrived > n_imu || scans[k].odom_arrived < op ||
        scans[k].odom_arrived > n_odom)
      B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_lidar_undistortion_node: arrival counts decrease or exceed their log");
  }
  if (n_scans == 0) return B2S_OK;
  if (b2s_status st = open_device(device)) return st;
  // a fresh node of one recording through the handle's path, its rows indexed by the corrected scan
  b2s_deskew_node h;
  h.st.s = reinterpret_cast<cudaStream_t>(cuda_stream);
  const b2s_deskew_laser laser = {angle_min, angle_increment, n_beams, use_imu, use_odom, 0};
  std::vector<double2> cs;
  nodes_init(h, 1, &laser, device, cs);
  AsyncBuf<double2> d_cs(h.st);
  B2S_CUDA_CHECK(d_cs.alloc(cs.size()));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_cs, cs.data(), cs.size() * sizeof(double2), cudaMemcpyHostToDevice, h.st));
  h.angle_cs = d_cs;
  const std::vector<long long> scan_first = {0, n_scans}, imu_first = {0, n_imu}, odom_first = {0, n_odom};
  if (b2s_status st = nodes_process(h, 1, &n_scans, scans, ranges, imu, odom, scan_first, imu_first, odom_first, out_status,
                                    out_state, out_xyz))
    return st;
  // scan n_scans - 1 is popped by the callback of a scan that never comes (CacheLaserScan, :145-150)
  out_status[n_scans - 1] = B2S_DESKEW_HELD;
  if (out_state) std::memset(&out_state[n_scans - 1], 0, sizeof(b2s_deskew_scan));
  return B2S_OK;
}

b2s_status b2s_deskew_node_create(int batch, const b2s_deskew_laser *lasers, int device, void *cuda_stream,
                                  b2s_deskew_node **out) {
  B2S_NVTX("LidarUndistortion nodes create");
  if (!out || !lasers || batch < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_create: null argument or batch < 1");
  *out = nullptr;
  for (int b = 0; b < batch; b++)
    if (lasers[b].n_beams < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_create: a laser without beams");
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<b2s_deskew_node> h(new (std::nothrow) b2s_deskew_node());
  if (!h) B2S_FAIL(B2S_ERR_CUDA, "b2s_deskew_node_create: out of host memory");
  B2S_CUDA_CHECK(h->st.init(cuda_stream));
  std::vector<double2> cs;
  nodes_init(*h, batch, lasers, device, cs);
  B2S_CUDA_CHECK(h->angles.reserve(cs.size()));
  B2S_CUDA_CHECK(h->held.reserve(cs.size()));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->angles, cs.data(), cs.size() * sizeof(double2), cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  h->angle_cs = h->angles;
  *out = h.release();
  return B2S_OK;
}

void b2s_deskew_node_destroy(b2s_deskew_node *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->st);
  delete h;
}

b2s_status b2s_deskew_node_reset(b2s_deskew_node *h, int recording) {
  if (!h || recording < -1 || recording >= h->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_reset: invalid argument");
  if (h->failed) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_deskew_node_reset: an earlier call failed on the device; destroy the handle");
  const int lo = recording < 0 ? 0 : recording, hi = recording < 0 ? h->batch : recording + 1;
  for (int b = lo; b < hi; b++) h->rec[b] = NodeState();
  return B2S_OK;
}

b2s_status b2s_deskew_node_process(b2s_deskew_node *h, const int32_t *n_scans, const b2s_deskew_node_scan *scans,
                                   const float *ranges, const int32_t *n_imu, const b2s_imu_msg *imu, const int32_t *n_odom,
                                   const b2s_odom_msg *odom, int32_t *out_status, b2s_deskew_scan *out_state,
                                   float *out_xyz) {
  B2S_NVTX("LidarUndistortion nodes process");
  if (!h) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_deskew_node_process: null handle");
  if (h->failed)
    B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_deskew_node_process: an earlier call failed on the device; destroy the handle");
  std::vector<long long> scan_first, imu_first, odom_first;
  if (b2s_status st = nodes_check(*h, n_scans, scans, ranges, n_imu, imu, n_odom, odom, out_status, out_xyz, scan_first,
                                  imu_first, odom_first))
    return st;
  if (cudaSetDevice(h->device) != cudaSuccess) {
    h->failed = true;
    B2S_FAIL(B2S_ERR_CUDA, "b2s_deskew_node_process: cudaSetDevice failed");
  }
  const b2s_status st = nodes_process(*h, 0, n_scans, scans, ranges, imu, odom, scan_first, imu_first, odom_first,
                                      out_status, out_state, out_xyz);
  if (st != B2S_OK) h->failed = true;
  return st;
}

}  // extern "C"
