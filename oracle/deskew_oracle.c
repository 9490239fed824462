/* TEST INFRASTRUCTURE — CPU restatement of lesson5's motion de-skew (LidarUndistortion, lesson5/src/lidar_undistortion.cc).
 * Pinned bit for bit to the unmodified node (oracle/ref_lesson5.cpp, tests/test_deskew_reference.py) except for the
 * arithmetic that lives in third-party headers not in the reference tree — pcl::getTransformation (PCL 1.8
 * common/impl/eigen.hpp) and Eigen 3.3 Affine3f inverse / product — which is restated here from their published
 * algorithms, and the same way in the node's stand-ins; whether PCL's unqualified cos / sin resolve to the float or the
 * double C functions cannot be checked (the double ones, rounded to float, are used, as the lesson4 headers were found
 * to do).
 *   orc_deskew_integrate_imu   PruneImuDeque's angle integration        (lidar_undistortion.cc:196-238)
 *   orc_deskew_odom_increment  PruneOdomDeque's odometry increment      (:296-333)
 *   orc_deskew_scan            CorrectLaserScan                          (:339-393) with ComputeRotation (:396-430) and
 *                              ComputePosition (:433-445) */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct {
  double time_start, time_increment;
  float range_min, range_max;
  int32_t use_imu, use_odom;
  int32_t imu_last, pad_;
  double odom_start_time, odom_end_time;
  float odom_incre[3];
  float pad2_;
} orc_deskew_scan_info;

typedef struct { float m[3][3]; float t[3]; } affine3f;

static float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); } /* Eigen's unrolled 3-term redux */

/* pcl::getTransformation (common/impl/eigen.hpp) */
static affine3f get_transformation(float x, float y, float z, float roll, float pitch, float yaw) {
  const float A = (float)cos((double)yaw), B = (float)sin((double)yaw), C = (float)cos((double)pitch), D = (float)sin((double)pitch),
              E = (float)cos((double)roll), F = (float)sin((double)roll), DE = D * E, DF = D * F;
  affine3f t;
  t.m[0][0] = A * C; t.m[0][1] = A * DF - B * E; t.m[0][2] = B * F + A * DE; t.t[0] = x;
  t.m[1][0] = B * C; t.m[1][1] = A * E + B * DF; t.m[1][2] = B * DE - A * F; t.t[1] = y;
  t.m[2][0] = -D;    t.m[2][1] = C * F;          t.m[2][2] = C * E;          t.t[2] = z;
  return t;
}

static float cofactor(const float m[3][3], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
}

/* Transform<float,3,Affine>::inverse(): linear part by Eigen's compute_inverse_size3 (cofactors), t' = -(L^-1 t) */
static affine3f affine_inverse(const affine3f *a) {
  affine3f r;
  const float c0 = cofactor(a->m, 0, 0), c1 = cofactor(a->m, 1, 0), c2 = cofactor(a->m, 2, 0);
  const float det = sum3(c0 * a->m[0][0], c1 * a->m[1][0], c2 * a->m[2][0]);
  const float invdet = 1.0f / det;
  r.m[0][0] = c0 * invdet; r.m[0][1] = c1 * invdet; r.m[0][2] = c2 * invdet;
  r.m[1][0] = cofactor(a->m, 0, 1) * invdet; r.m[1][1] = cofactor(a->m, 1, 1) * invdet; r.m[1][2] = cofactor(a->m, 2, 1) * invdet;
  r.m[2][0] = cofactor(a->m, 0, 2) * invdet; r.m[2][1] = cofactor(a->m, 1, 2) * invdet; r.m[2][2] = cofactor(a->m, 2, 2) * invdet;
  for (int i = 0; i < 3; i++) r.t[i] = -sum3(r.m[i][0] * a->t[0], r.m[i][1] * a->t[1], r.m[i][2] * a->t[2]);
  return r;
}

/* Affine * Affine: linear = L1 L2, translation = L1 t2 + t1 */
static affine3f affine_mul(const affine3f *a, const affine3f *b) {
  affine3f r;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) r.m[i][j] = sum3(a->m[i][0] * b->m[0][j], a->m[i][1] * b->m[1][j], a->m[i][2] * b->m[2][j]);
    r.t[i] = sum3(a->m[i][0] * b->t[0], a->m[i][1] * b->t[1], a->m[i][2] * b->t[2]) + a->t[i];
  }
  return r;
}

int32_t orc_deskew_integrate_imu(int n_imu, const double *stamp, const double *ang_vel, double scan_start, double scan_end,
                                 int cap, double *imu_time, double *rx, double *ry, double *rz) {
  int idx = 0;
  for (int i = 0; i < cap; i++) imu_time[i] = rx[i] = ry[i] = rz[i] = 0.0;
  for (int i = 0; i < n_imu; i++) {
    const double t = stamp[i];
    if (t < scan_start) {
      if (idx == 0) { rx[0] = ry[0] = rz[0] = 0.0; imu_time[0] = t; ++idx; }
      continue;
    }
    if (t > scan_end) break;
    if (idx == 0 || idx >= cap) return -2;  /* the node would index imu_time_[-1] / overflow its queue: caller error */
    const double dt = t - imu_time[idx - 1];
    rx[idx] = rx[idx - 1] + ang_vel[3 * i] * dt;
    ry[idx] = ry[idx - 1] + ang_vel[3 * i + 1] * dt;
    rz[idx] = rz[idx - 1] + ang_vel[3 * i + 2] * dt;
    imu_time[idx] = t;
    ++idx;
  }
  return idx - 1;
}

void orc_deskew_odom_increment(const double start[6], const double end[6], float out[3]) {
  const affine3f b = get_transformation((float)start[0], (float)start[1], (float)start[2], (float)start[3], (float)start[4], (float)start[5]);
  const affine3f e = get_transformation((float)end[0], (float)end[1], (float)end[2], (float)end[3], (float)end[4], (float)end[5]);
  const affine3f bi = affine_inverse(&b);
  const affine3f bt = affine_mul(&bi, &e);
  out[0] = bt.t[0]; out[1] = bt.t[1]; out[2] = bt.t[2];  /* pcl::getTranslationAndEulerAngles: x, y, z = t(0..2, 3) */
}

static void compute_rotation(const orc_deskew_scan_info *s, const double *imu_time, const double *rx, const double *ry,
                             const double *rz, double t, float *ox, float *oy, float *oz) {
  int front = 0;
  while (front < s->imu_last) {
    if (t < imu_time[front]) break;
    ++front;
  }
  if (t > imu_time[front] || front == 0) {
    *ox = (float)rx[front]; *oy = (float)ry[front]; *oz = (float)rz[front];
  } else {
    const int back = front - 1;
    const double rf = (t - imu_time[back]) / (imu_time[front] - imu_time[back]);
    const double rb = (imu_time[front] - t) / (imu_time[front] - imu_time[back]);
    *ox = (float)(rx[front] * rf + rx[back] * rb);
    *oy = (float)(ry[front] * rf + ry[back] * rb);
    *oz = (float)(rz[front] * rf + rz[back] * rb);
  }
}

void orc_deskew_scan(int n_beams, const float *ranges, double angle_min, double angle_increment, const orc_deskew_scan_info *s,
                     const double *imu_time, const double *rx, const double *ry, const double *rz, float *out_xyz) {
  int first = 1;
  affine3f start_inv;
  memset(&start_inv, 0, sizeof(start_inv));
  for (int i = 0; i < n_beams; i++) {
    float *o = out_xyz + 3 * i;
    o[0] = o[1] = o[2] = 0.0f;  /* the cloud is cleared and resized per scan: skipped points stay default */
    const float r = ranges[i];
    if (!isfinite(r) || r < s->range_min || r > s->range_max) continue;
    const double t = s->time_start + i * s->time_increment;
    /* CreateAngleCache (:162-174): float fields and an unsigned index, so the angle is summed in float */
    const float step = (float)(unsigned)i * (float)angle_increment;
    const double angle = (float)angle_min + step;
    const double px = r * cos(angle), py = r * sin(angle), pz = 1.0;
    float rotx = 0, roty = 0, rotz = 0, posx = 0, posy = 0, posz = 0;
    if (s->use_imu) compute_rotation(s, imu_time, rx, ry, rz, t, &rotx, &roty, &rotz);
    if (s->use_odom) {
      const double ratio = (t - s->odom_start_time) / (s->odom_end_time - s->odom_start_time);
      posx = (float)(s->odom_incre[0] * ratio); posy = (float)(s->odom_incre[1] * ratio); posz = (float)(s->odom_incre[2] * ratio);
    }
    const affine3f fin = get_transformation(posx, posy, posz, rotx, roty, rotz);
    if (first) { start_inv = affine_inverse(&fin); first = 0; }
    const affine3f bt = affine_mul(&start_inv, &fin);
    o[0] = (float)(bt.m[0][0] * px + bt.m[0][1] * py + bt.m[0][2] * pz + bt.t[0]);
    o[1] = (float)(bt.m[1][0] * px + bt.m[1][1] * py + bt.m[1][2] * pz + bt.t[1]);
    o[2] = (float)(bt.m[2][0] * px + bt.m[2][1] * py + bt.m[2][2] * pz + bt.t[2]);
  }
}
