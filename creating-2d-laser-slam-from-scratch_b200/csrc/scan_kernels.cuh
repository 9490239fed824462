// Kernels shared by the Karto matcher (K1) and the Karto occupancy grid (K2c).  `static`: each translation unit
// gets its own copy, the library exports nothing from here.
#pragma once
#include "common.cuh"

namespace b2s {

// ----------------------------------------------------------------------------------------------
// k_scan_points: LocalizedRangeScan::Update unfiltered points (Karto.h:5362-5404) and, optionally, the
// scan-local points of GridIndexLookup::ComputeOffsets (Karto.h:6423-6434, Transform::InverseTransformPose
// Karto.h:2894-2901).  One block per scan.
// ----------------------------------------------------------------------------------------------
// `src` (may be NULL): row of `ranges` scan b reads (a scan pool shared by many base sets); NULL = row b.
// The float overload reads float32 readings widened to double (the Karto node's map pool), which is exact.
template <class R>
static __device__ __forceinline__ void scan_points_block(const R *__restrict__ ranges, const double *__restrict__ poses,
                                                         const b2s_laser &l, double *__restrict__ sensor,
                                                         double *__restrict__ pts, double *__restrict__ local,
                                                         const int32_t *__restrict__ src) {
  const int b = blockIdx.x;
  const size_t row = src ? (size_t)src[b] : (size_t)b;
  const int n = l.n_readings;
  __shared__ double sp[3];
  __shared__ double inv[6];
  __shared__ double tr[3];
  if (threadIdx.x == 0) {
    double robot[3] = {poses[3 * b], poses[3 * b + 1], poses[3 * b + 2]};
    double out[3];
    sensor_pose_of(robot, l.offset_pose, out);
    sp[0] = out[0]; sp[1] = out[1]; sp[2] = out[2];
    if (sensor) { sensor[3 * b] = out[0]; sensor[3 * b + 1] = out[1]; sensor[3 * b + 2] = out[2]; }
    if (out[0] == 0.0 && out[1] == 0.0 && out[2] == 0.0) {
      inv[0] = 1; inv[1] = 0; inv[2] = 0; inv[3] = 0; inv[4] = 1; inv[5] = 0;
      tr[0] = tr[1] = tr[2] = 0;
    } else {
      double radians = 0.0 - out[2];
      double c = cos(radians), s = sin(radians), omc = 1.0 - c;
      inv[0] = 0.0 * omc + c;
      inv[1] = 0.0 * 0.0 * omc - 1.0 * s;
      inv[2] = 0.0 * 1.0 * omc + 0.0 * s;
      inv[3] = 0.0 * 0.0 * omc + 1.0 * s;
      inv[4] = 0.0 * omc + c;
      inv[5] = 0.0 * 1.0 * omc - 0.0 * s;
      tr[0] = out[0]; tr[1] = out[1]; tr[2] = out[2] - 0.0;
    }
  }
  __syncthreads();
  const double dh = normalize_angle(0.0 - tr[2]);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double r = (double)ranges[row * n + i];
    double angle = sp[2] + l.min_angle + (double)(uint32_t)i * l.angular_resolution;
    double x = sp[0] + (r * cos(angle));
    double y = sp[1] + (r * sin(angle));
    pts[((size_t)b * n + i) * 2] = x;
    pts[((size_t)b * n + i) * 2 + 1] = y;
    if (local) {
      double dx = x - tr[0], dy = y - tr[1];
      local[((size_t)b * n + i) * 2] = inv[0] * dx + inv[1] * dy + inv[2] * dh;
      local[((size_t)b * n + i) * 2 + 1] = inv[3] * dx + inv[4] * dy + inv[5] * dh;
    }
  }
}
static __global__ void k_scan_points(const double *__restrict__ ranges, const double *__restrict__ poses, b2s_laser l,
                                     double *__restrict__ sensor, double *__restrict__ pts, double *__restrict__ local,
                                     const int32_t *__restrict__ src) {
  scan_points_block(ranges, poses, l, sensor, pts, local, src);
}
static __global__ void k_scan_points(const float *__restrict__ ranges, const double *__restrict__ poses, b2s_laser l,
                                     double *__restrict__ sensor, double *__restrict__ pts, double *__restrict__ local,
                                     const int32_t *__restrict__ src) {
  scan_points_block(ranges, poses, l, sensor, pts, local, src);
}


}  // namespace b2s
