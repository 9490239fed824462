// lesson5 motion de-skew as a device pre-stage (SURVEY.md §8(f).4): LidarUndistortion::CorrectLaserScan
// (lesson5/src/lidar_undistortion.cc:339-393) for a BATCH of LaserScans — every beam of every scan is one thread — with
// ComputeRotation (:396-430: linear interpolation in the integrated IMU angles) and ComputePosition (:433-445: linear
// in the odometry increment).  The per-scan preparation the node does under its queue locks is provided as host
// functions with the node's arithmetic: PruneImuDeque's angle integration (:196-238) and PruneOdomDeque's odometry
// increment (:296-333).  b2s_lidar_undistortion_node runs the whole node over a recording: the callbacks and both queue
// prunes on the host, then one CTA per published scan that integrates the scan's IMU queue into shared memory and
// corrects its beams.
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

// ---- the node over a recording (b2s_lidar_undistortion_node) ----

// a published scan: its output row, the pruned IMU queue as [imu_lo, imu_lo + imu_n) of the log, and its scan end
struct NodeRow {
  int32_t row, imu_lo, imu_n, reserved;
  double scan_end;
};

// One CTA per published scan (grid x, up to 2^31 - 1 scans).  Thread 0 integrates the scan's IMU queue from the log
// into shared memory, [4][stride] doubles with stride the call's largest table; entry 0 is zeroed first, so that
// imu_last = -1 (no message before the scan start) takes rotation 0 as the node's reset table gives.  Then the CTA finds
// the first valid reading, thread 0 inverts its pose once, and the CTA walks all beams.
constexpr int NODE_THREADS = 256;
__global__ void __launch_bounds__(NODE_THREADS)
    k_deskew_node(const float *__restrict__ ranges, int n_beams, const double2 *__restrict__ angle_cs,
                  const NodeRow *__restrict__ rows, const b2s_deskew_scan *__restrict__ states,
                  const double *__restrict__ log_t, const double *__restrict__ log_x, const double *__restrict__ log_y,
                  const double *__restrict__ log_z, int stride, float *__restrict__ out_xyz) {
  extern __shared__ double s_tab[];
  double *it = s_tab, *rx = s_tab + stride, *ry = rx + stride, *rz = ry + stride;
  const NodeRow w = rows[blockIdx.x];
  const b2s_deskew_scan s = states[blockIdx.x];
  const float *r = ranges + (size_t)w.row * n_beams;
  float *out = out_xyz + (size_t)w.row * n_beams * 3;
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
    deskew_beam(s, s_inv, it, rx, ry, rz, i, range, angle_cs[i], o);
  }
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

  // ---- the callbacks, on the host: statuses, per-scan states and the IMU queue of every published scan
  std::vector<double> imu_t(use_imu ? n_imu : 0), odom_t(use_odom ? n_odom : 0);
  for (size_t i = 0; i < imu_t.size(); i++) imu_t[i] = ros_time_to_sec(imu[i].sec, imu[i].nsec);
  for (size_t i = 0; i < odom_t.size(); i++) odom_t[i] = ros_time_to_sec(odom[i].sec, odom[i].nsec);
  const double scan_count = (double)n_beams;  // scan_count_, a double member, from the first scan (:136)
  std::vector<NodeRow> rows;
  std::vector<b2s_deskew_scan> states;
  int ilo = 0, olo = 0;              // fronts of the IMU and odometry queues in their logs
  int start_msg = -1, end_msg = -1;  // start_odom_msg_ / end_odom_msg_ (members): -1 is the default-constructed message
  int stride = 1;                    // the largest IMU table of a published scan
  for (int j = 0; j < n_scans; j++) {
    b2s_deskew_scan s;
    std::memset(&s, 0, sizeof s);
    int32_t status = B2S_DESKEW_PUBLISHED;
    NodeRow w = {j, 0, 0, 0, 0.0};
    [&] {
      if (j == n_scans - 1) {  // scan j is popped by the callback of scan j + 1 (CacheLaserScan, :145-150)
        status = B2S_DESKEW_HELD;
        return;
      }
      const b2s_deskew_node_scan &sc = scans[j], &next = scans[j + 1];
      const double start = ros_time_to_sec(sc.sec, sc.nsec), inc = sc.time_increment, end = start + inc * (scan_count - 1);
      w.scan_end = end;
      s.time_start = start;
      s.time_increment = inc;
      s.range_min = sc.range_min;
      s.range_max = sc.range_max;
      s.use_imu = use_imu != 0;
      s.use_odom = use_odom != 0;
      if (use_imu) {  // PruneImuDeque (:177-249)
        const int hi = next.imu_arrived;
        if (ilo == hi || imu_t[ilo] > start || imu_t[hi - 1] < end) {
          status = B2S_DESKEW_WAIT_IMU;
          return;
        }
        while (ilo < hi && imu_t[ilo] < start - 0.1) ++ilo;
        if (ilo == hi) {
          status = B2S_DESKEW_IMU_EMPTY;
          return;
        }
        w.imu_lo = ilo;
        w.imu_n = hi - ilo;
        s.imu_last = imu_table<false>(w.imu_n, imu_t.data() + ilo, nullptr, nullptr, nullptr, 0, start, end,
                                      IMU_QUEUE_LENGTH, nullptr, nullptr, nullptr, nullptr);
        if (s.imu_last == -2) status = B2S_DESKEW_UNDEFINED;  // the odometry queue is still pruned, as the node goes on
      }
      if (use_odom) {  // PruneOdomDeque (:252-336)
        const int hi = next.odom_arrived;
        if (olo == hi || odom_t[olo] > start || odom_t[hi - 1] < end) {
          if (status == B2S_DESKEW_PUBLISHED) status = B2S_DESKEW_WAIT_ODOM;
          return;
        }
        while (olo < hi && odom_t[olo] < start - 0.1) ++olo;
        if (olo == hi) {
          if (status == B2S_DESKEW_PUBLISHED) status = B2S_DESKEW_ODOM_EMPTY;
          return;
        }
        for (int i = olo; i < hi; i++) {
          if (odom_t[i] < start) {
            start_msg = i;
            continue;
          }
          if (odom_t[i] <= end)
            end_msg = i;
          else
            break;
        }
        const b2s_odom_msg none = {};
        double sp[6], ep[6];
        odom_pose(start_msg < 0 ? none : odom[start_msg], sp);
        odom_pose(end_msg < 0 ? none : odom[end_msg], ep);
        s.odom_start_time = start_msg < 0 ? 0.0 : odom_t[start_msg];
        s.odom_end_time = end_msg < 0 ? 0.0 : odom_t[end_msg];
        b2s_deskew_odom_increment(sp, ep, s.odom_incre);
      }
    }();
    out_status[j] = status;
    if (status == B2S_DESKEW_PUBLISHED || status == B2S_DESKEW_UNDEFINED) {
      if (out_state) out_state[j] = s;
    } else if (out_state) {
      std::memset(&out_state[j], 0, sizeof s);
    }
    if (status == B2S_DESKEW_PUBLISHED) {
      rows.push_back(w);
      states.push_back(s);
      if (use_imu) stride = std::max(stride, s.imu_last + 1);
    }
  }
  const size_t n_pub = rows.size(), nr = (size_t)n_scans * n_beams;
  if (n_pub == 0) {
    std::memset(out_xyz, 0, nr * 3 * sizeof(float));
    return B2S_OK;
  }

  // ---- one upload of the call's small inputs: beam angles (CreateAngleCache, :162-174, as b2s_lidar_undistort takes
  // them), the IMU log as SoA doubles, and the published scans
  const size_t n_log = use_imu ? (size_t)n_imu : 0;
  const size_t off_log = 2 * (size_t)n_beams, off_states = off_log + 4 * n_log;
  const size_t off_rows = off_states + n_pub * sizeof(b2s_deskew_scan) / sizeof(double);
  static_assert(sizeof(b2s_deskew_scan) % sizeof(double) == 0 && sizeof(NodeRow) % sizeof(double) == 0, "packing");
  std::vector<double> pack(off_rows + n_pub * sizeof(NodeRow) / sizeof(double));
  for (int i = 0; i < n_beams; i++) {
    const float step = (float)(unsigned)i * angle_increment;
    const double angle = angle_min + step;
    pack[2 * i] = cos(angle);
    pack[2 * i + 1] = sin(angle);
  }
  for (size_t i = 0; i < n_log; i++) {
    pack[off_log + i] = imu_t[i];
    for (int a = 0; a < 3; a++) pack[off_log + (a + 1) * n_log + i] = imu[i].angular_velocity[a];
  }
  std::memcpy(pack.data() + off_states, states.data(), n_pub * sizeof(b2s_deskew_scan));
  std::memcpy(pack.data() + off_rows, rows.data(), n_pub * sizeof(NodeRow));

  cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
  const size_t smem = 4 * sizeof(double) * (size_t)stride;  // at most 2000 entries: 64 000 bytes
  if (smem > 48 * 1024) B2S_CUDA_CHECK(raise_dyn_smem(k_deskew_node, smem));
  AsyncBuf<float> d_r(st), d_o(st);
  AsyncBuf<double> d_pack(st);
  B2S_CUDA_CHECK(d_r.alloc(nr));
  B2S_CUDA_CHECK(d_o.alloc(nr * 3));
  B2S_CUDA_CHECK(d_pack.alloc(pack.size()));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, nr * sizeof(float), cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_pack, pack.data(), pack.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  // rows the kernel does not write are zero bytes: one memset per run of unpublished scans
  for (size_t p = 0, next = 0; p <= n_pub; p++) {
    const size_t until = p < n_pub ? (size_t)rows[p].row : (size_t)n_scans;
    if (until > next)
      B2S_CUDA_CHECK(cudaMemsetAsync(d_o + next * n_beams * 3, 0, (until - next) * n_beams * 3 * sizeof(float), st));
    next = until + 1;
  }
  const double *log = d_pack + off_log;
  k_deskew_node<<<(unsigned)n_pub, NODE_THREADS, smem, st>>>(
      d_r, n_beams, reinterpret_cast<const double2 *>(static_cast<double *>(d_pack)),
      reinterpret_cast<const NodeRow *>(d_pack + off_rows), reinterpret_cast<const b2s_deskew_scan *>(d_pack + off_states),
      log, log + n_log, log + 2 * n_log, log + 3 * n_log, stride, d_o);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out_xyz, d_o, nr * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  return B2S_OK;
}

}  // extern "C"
