// lesson5 motion de-skew as a device pre-stage (SURVEY.md §8(f).4): LidarUndistortion::CorrectLaserScan
// (lesson5/src/lidar_undistortion.cc:339-393) for a BATCH of LaserScans — every beam of every scan is one thread — with
// ComputeRotation (:396-430: linear interpolation in the integrated IMU angles) and ComputePosition (:433-445: linear
// in the odometry increment).  The per-scan preparation the node does under its queue locks is provided as host
// functions with the node's arithmetic: PruneImuDeque's angle integration (:196-238) and PruneOdomDeque's odometry
// increment (:296-333).
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
  const double2 cs = angle_cs[i];  // a_cos_[i], a_sin_[i]
  const double px = range * cs.x, py = range * cs.y, pz = 1.0;
  const Affine3f bt = affine_mul(s_inv, pose_at(s, it, rx, ry, rz, i));
  o[0] = (float)(bt.m[0][0] * px + bt.m[0][1] * py + bt.m[0][2] * pz + bt.t[0]);
  o[1] = (float)(bt.m[1][0] * px + bt.m[1][1] * py + bt.m[1][2] * pz + bt.t[1]);
  o[2] = (float)(bt.m[2][0] * px + bt.m[2][1] * py + bt.m[2][2] * pz + bt.t[2]);
}

}  // namespace

extern "C" {

int32_t b2s_deskew_integrate_imu(int n_imu, const double *stamp, const double *angular_velocity, double scan_time_start,
                                 double scan_time_end, int capacity, double *imu_time, double *rot_x, double *rot_y,
                                 double *rot_z) {
  if (n_imu < 0 || capacity < 1 || !imu_time || !rot_x || !rot_y || !rot_z || (n_imu > 0 && (!stamp || !angular_velocity))) return -2;
  for (int i = 0; i < capacity; i++) imu_time[i] = rot_x[i] = rot_y[i] = rot_z[i] = 0.0;  // ResetParameters (:66-74)
  int idx = 0;
  for (int i = 0; i < n_imu; i++) {
    const double t = stamp[i];
    if (t < scan_time_start) {
      if (idx == 0) {
        rot_x[0] = rot_y[0] = rot_z[0] = 0.0;
        imu_time[0] = t;
        ++idx;
      }
      continue;
    }
    if (t > scan_time_end) break;
    if (idx == 0 || idx >= capacity) return -2;  // the node would read imu_time_[-1] / overrun its queue
    const double dt = t - imu_time[idx - 1];
    rot_x[idx] = rot_x[idx - 1] + angular_velocity[3 * i] * dt;
    rot_y[idx] = rot_y[idx - 1] + angular_velocity[3 * i + 1] * dt;
    rot_z[idx] = rot_z[idx - 1] + angular_velocity[3 * i + 2] * dt;
    imu_time[idx] = t;
    ++idx;
  }
  return idx - 1;
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

}  // extern "C"
