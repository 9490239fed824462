/*
 * pcl_icp_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the lesson2 node (reference/lesson2/src/scan_match_icp.cc):
 *   orc_pcl_scan_to_cloud  ConvertScan2PointCloud (:89-130): one pcl::PointXYZ per reading, invalid readings left at
 *                          the default (0, 0, 0) and kept in the cloud (width = ranges.size(), is_dense = true)
 *   orc_pcl_icp_align      ScanMatchWithICP (:135-164): a default-constructed
 *                          pcl::IterativeClosestPoint<PointXYZ, PointXYZ>, source = previous cloud, target = current
 *                          cloud, align() without a guess; hasConverged(), getFinalTransformation() turned into
 *                          (x, y, yaw) by pcl::getTranslationAndEulerAngles, getFitnessScore()
 *
 * PARITY UNPINNED.  PCL (1.8, the ROS Kinetic package install_dependence.sh pulls) is third-party code absent from the
 * reference tree and from this image.  Every step below restates its published behaviour; the choices that could not be
 * checked against PCL itself are listed in DESIGN.md §2:
 *   - the node's unqualified cos / sin of a float angle are taken as the float functions (cosf / sinf of the C library);
 *   - nearest neighbours are exact (KdTreeFLANN searches exactly); among equidistant targets the lowest index wins;
 *   - the SVD rigid fit of planar points is its 2-D closed form, with the sums in a fixed order: every reduction runs
 *     over PCL_ICP_LANES lanes (lane t takes points t, t + lanes, ... in order), then a tree inside each 32-lane group,
 *     then a tree over the groups — the order the device kernel reduces in;
 *   - DefaultConvergenceCriteria starts every align() afresh (previous MSE = DBL_MAX).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h"

#define PCL_ICP_LANES 256
#define PCL_ICP_GROUPS (PCL_ICP_LANES / 32)

/* tree over the lanes: inside each 32-lane group lane l += lane l + d for d = 16, 8, 4, 2, 1; then group g += group
 * g + d for d = 4, 2, 1.  The values of one level are read before that level writes them. */
#define DEFINE_TREE(name, T)                                                              \
  static T name(T *v) {                                                                   \
    T g[PCL_ICP_GROUPS];                                                                  \
    for (int w = 0; w < PCL_ICP_GROUPS; w++) {                                            \
      T *x = v + 32 * w;                                                                  \
      for (int d = 16; d > 0; d >>= 1)                                                    \
        for (int l = 0; l < d; l++) x[l] += x[l + d];                                     \
      g[w] = x[0];                                                                        \
    }                                                                                     \
    for (int d = PCL_ICP_GROUPS / 2; d > 0; d >>= 1)                                      \
      for (int k = 0; k < d; k++) g[k] += g[k + d];                                       \
    return g[0];                                                                          \
  }
DEFINE_TREE(tree_f, float)
DEFINE_TREE(tree_d, double)

int orc_pcl_scan_to_cloud(int n, const float *ranges, float angle_min, float angle_increment, float range_min,
                          float range_max, int drop_invalid, float *xy) {
  int m = 0;
  for (int i = 0; i < n; i++) {
    const float range = ranges[i];
    const int valid = isfinite(range) && range > range_min && range < range_max; /* :104-109 */
    float x = 0.0f, y = 0.0f;
    if (valid) {
      const float angle = angle_min + (float)(unsigned)i * angle_increment; /* :112, float */
      x = range * cosf(angle);
      y = range * sinf(angle);
    }
    if (valid || !drop_invalid) { xy[2 * m] = x; xy[2 * m + 1] = y; m++; }
  }
  return m;
}

/* exact nearest target of q: squared distance dx*dx + dy*dy in float, first (lowest) index among equal distances;
 * -1 when no target is at a finite distance */
static int nearest(const float *tgt, int nt, float qx, float qy, float *dist) {
  int bj = -1;
  float bd = INFINITY;
  for (int j = 0; j < nt; j++) {
    const float dx = qx - tgt[2 * j], dy = qy - tgt[2 * j + 1];
    const float d = dx * dx + dy * dy;
    if (d < bd) { bd = d; bj = j; }
  }
  *dist = bd;
  return bj;
}

/* pcl::transformPointCloud with a planar Matrix4f (rows f00 f01 tx / f10 f11 ty): x' = (f00 x + f01 y) + tx */
static void apply(const float f[6], float x, float y, float *ox, float *oy) {
  *ox = (f[0] * x + f[1] * y) + f[2];
  *oy = (f[3] * x + f[4] * y) + f[5];
}

/* src [ns][2], tgt [nt][2]; guess (x, y, yaw) or NULL for align()'s identity */
void orc_pcl_icp_align(const b2s_pcl_icp_params *P, int ns, const float *src, int nt, const float *tgt,
                       const float *guess, b2s_pcl_icp_result *out) {
  float *cur = malloc(sizeof(float) * 2 * (ns > 0 ? ns : 1));
  int *nn = malloc(sizeof(int) * (ns > 0 ? ns : 1));
  float *nd = malloc(sizeof(float) * (ns > 0 ? ns : 1));
  float fl[5][PCL_ICP_LANES];
  double dl[PCL_ICP_LANES];
  int il[PCL_ICP_LANES];
  const double max_d2 = P->max_correspondence_distance * P->max_correspondence_distance;
  const double rot_thr = 1.0 - P->transformation_epsilon, trans_thr = P->transformation_epsilon;

  /* final_transformation_ = guess; the source is transformed first only if the guess is not the identity */
  float f[6] = {1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f};
  if (guess) {
    const float c = cosf(guess[2]), s = sinf(guess[2]);
    f[0] = c; f[1] = -s; f[2] = guess[0]; f[3] = s; f[4] = c; f[5] = guess[1];
  }
  const int identity = f[0] == 1.0f && f[1] == 0.0f && f[2] == 0.0f && f[3] == 0.0f && f[4] == 1.0f && f[5] == 0.0f;
  for (int i = 0; i < ns; i++) {
    if (identity) { cur[2 * i] = src[2 * i]; cur[2 * i + 1] = src[2 * i + 1]; }
    else apply(f, src[2 * i], src[2 * i + 1], &cur[2 * i], &cur[2 * i + 1]);
  }

  double prev_mse = DBL_MAX;
  int iterations = 0, converged = 0, n_corr = 0;
  for (;;) {
    /* correspondences: the nearest target of every source point, dropped beyond the distance threshold */
    for (int i = 0; i < ns; i++) {
      float d;
      const int j = nearest(tgt, nt, cur[2 * i], cur[2 * i + 1], &d);
      nn[i] = (j >= 0 && !((double)d > max_d2)) ? j : -1;
      nd[i] = d;
    }
    /* centroids */
    for (int t = 0; t < PCL_ICP_LANES; t++) {
      int cnt = 0;
      float spx = 0.0f, spy = 0.0f, sqx = 0.0f, sqy = 0.0f;
      for (int i = t; i < ns; i += PCL_ICP_LANES) {
        if (nn[i] < 0) continue;
        cnt++;
        spx += cur[2 * i]; spy += cur[2 * i + 1];
        sqx += tgt[2 * nn[i]]; sqy += tgt[2 * nn[i] + 1];
      }
      il[t] = cnt; fl[0][t] = spx; fl[1][t] = spy; fl[2][t] = sqx; fl[3][t] = sqy;
    }
    int count = 0;
    for (int t = 0; t < PCL_ICP_LANES; t++) count += il[t];
    n_corr = count;
    if (count < 3) { converged = 0; break; } /* min_number_correspondences_ */
    const float inv_n = 1.0f / (float)count;
    const float cpx = tree_f(fl[0]) * inv_n, cpy = tree_f(fl[1]) * inv_n;
    const float cqx = tree_f(fl[2]) * inv_n, cqy = tree_f(fl[3]) * inv_n;
    /* cross-covariance S = sum (p - cp)(q - cq)^T and the correspondence MSE */
    for (int t = 0; t < PCL_ICP_LANES; t++) {
      float sxx = 0.0f, sxy = 0.0f, syx = 0.0f, syy = 0.0f;
      double mse = 0.0;
      for (int i = t; i < ns; i += PCL_ICP_LANES) {
        if (nn[i] < 0) continue;
        const float px = cur[2 * i] - cpx, py = cur[2 * i + 1] - cpy;
        const float qx = tgt[2 * nn[i]] - cqx, qy = tgt[2 * nn[i] + 1] - cqy;
        sxx += px * qx; sxy += px * qy; syx += py * qx; syy += py * qy;
        mse += (double)nd[i];
      }
      fl[0][t] = sxx; fl[1][t] = sxy; fl[2][t] = syx; fl[3][t] = syy; dl[t] = mse;
    }
    const float sxx = tree_f(fl[0]), sxy = tree_f(fl[1]), syx = tree_f(fl[2]), syy = tree_f(fl[3]);
    const double mse = tree_d(dl) / (double)count;
    /* rigid increment: R = [[a, -b], [b, a]] / sqrt(a^2 + b^2), t = cq - R cp */
    const float a = sxx + syy, b = sxy - syx, h2 = a * a + b * b;
    float c = 1.0f, s = 0.0f;
    if (h2 != 0.0f) {
      const float h = sqrtf(h2);
      c = a / h; s = b / h;
    }
    const float tx = cqx - (c * cpx - s * cpy), ty = cqy - (s * cpx + c * cpy);
    /* transform the working cloud by the increment; final = increment * final */
    for (int i = 0; i < ns; i++) {
      const float x = cur[2 * i], y = cur[2 * i + 1];
      cur[2 * i] = (c * x - s * y) + tx;
      cur[2 * i + 1] = (s * x + c * y) + ty;
    }
    const float g[6] = {c * f[0] - s * f[3], c * f[1] - s * f[4], (c * f[2] - s * f[5]) + tx,
                        s * f[0] + c * f[3], s * f[1] + c * f[4], (s * f[2] + c * f[5]) + ty};
    memcpy(f, g, sizeof(g));
    ++iterations;
    /* DefaultConvergenceCriteria::hasConverged */
    if (iterations >= P->max_iterations) { converged = 1; break; } /* failure_after_max_iter_ = false */
    const double cos_angle = 0.5 * (double)(((c + c) + 1.0f) - 1.0f);
    const double translation_sqr = (double)((tx * tx + ty * ty) + 0.0f * 0.0f);
    if (cos_angle >= rot_thr && translation_sqr <= trans_thr) { converged = 1; break; }
    if (fabs(mse - prev_mse) < 1e-12) { converged = 1; break; }
    if (fabs(mse - prev_mse) / prev_mse < P->euclidean_fitness_epsilon) { converged = 1; break; }
    prev_mse = mse;
  }

  /* getFitnessScore(): the original source under the final transform, nearest target distance, averaged */
  for (int t = 0; t < PCL_ICP_LANES; t++) {
    double sum = 0.0;
    int nr = 0;
    for (int i = t; i < ns; i += PCL_ICP_LANES) {
      float x, y, d;
      apply(f, src[2 * i], src[2 * i + 1], &x, &y);
      if (nearest(tgt, nt, x, y, &d) >= 0 && (double)d <= DBL_MAX) { sum += (double)d; nr++; }
    }
    dl[t] = sum; il[t] = nr;
  }
  int nr = 0;
  for (int t = 0; t < PCL_ICP_LANES; t++) nr += il[t];
  const double fit = tree_d(dl);
  out->x[0] = f[2];
  out->x[1] = f[5];
  out->x[2] = atan2f(f[3], f[0]); /* pcl::getTranslationAndEulerAngles: yaw = atan2(t(1,0), t(0,0)) */
  out->converged = converged;
  out->iterations = iterations;
  out->n_correspondences = n_corr;
  out->fitness_score = nr > 0 ? fit / (double)nr : DBL_MAX;
  free(cur); free(nn); free(nd);
}
