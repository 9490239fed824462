/*
 * hector_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * Scalar C restatement of the lesson4 Hector grid map (K2a) and its Gauss-Newton scan matcher (K3 in-tree
 * analogue), paths relative to reference/lesson4/include/lesson4/hector_mapping:
 *   GridMapBase ctor / setMapTransformation / getMapCoordsPose / getWorldCoordsPose   map/GridMapBase.h:54-66, 238-286
 *   MapDimensionProperties::setMapCellDims (mapLimitsf = dims - 2)                   map/MapDimensionProperties.h:61-70
 *   LogOddsCell / GridMapLogOddsFunctions                                            map/GridMapLogOdds.h:37-161
 *   OccGridMapBase::updateByScan / updateLineBresenhami / bresenham2D / CellFree/Occ map/OccGridMapBase.h:118-168, 220-330
 *   OccGridMapUtil::getCompleteHessianDerivs / interpMapValueWithDerivatives         map/OccGridMapUtil.h:77-228, 437-440
 *   ScanMatcher::matchData / estimateTransformationLogLh                             matcher/ScanMatcher.h:60-141
 *   util::sign, util::normalize_angle                                               util/UtilFunctions.h:36-58
 *
 * PINNED (was "unpinned" until a way to execute the reference was found): Eigen is not installed in this image, so the
 * reference headers are compiled UNMODIFIED against a minimal stand-in for the fixed-size Eigen types they use
 * (oracle/shim/Eigen/mini_eigen.h; oracle/ref_hector.cpp -> oracle/_ref/libhector_ref.so).  This file agrees with that
 * build bit for bit — update indices, float32 log-odds, Gauss-Newton poses and Hessians, whole HectorSlamProcessor
 * streams (tests/test_oracle_hector_reference.py) — and with the golden vectors it produced (tests/golden/hector.npz).
 * What remains an assumption is only the stand-in's reading of Eigen's fixed-size primitives (listed in its header:
 * Translation*Rotation2D -> x' = (c*x + (-s)*y) + tx in float32 without FMA; AlignedScaling*Translation -> linear
 * diag(s,s), translation s*off; float -> int casts truncate; Affine / Matrix3f inverse in cofactor/determinant form;
 * 3-term sums as a0 + (a1 + a2)).  The live comparison found and fixed one slip of the restatement
 * (normalize_angle's `a -= 2.0f*M_PI` is evaluated in double).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

typedef struct {
  int size_x, size_y;
  float cell_length, scale_to_map;
  float off_x, off_y;          /* topLeftOffset passed to the GridMap ctor */
  float tw_lin, tw_tx, tw_ty;  /* mapTworld:  map = (tw_lin * w) + tw_t */
  float wt_lin, wt_tx, wt_ty;  /* worldTmap = mapTworld.inverse() */
  float log_odds_free, log_odds_occ;
  int curr_update_index;       /* currUpdateIndex (OccGridMapBase.h:50) */
  float *log_odds;
  int32_t *update_index;
} orc_hmap;

static float prob_to_log_odds(float prob) { /* GridMapLogOdds.h:153-157 */
  float odds = prob / (1.0f - prob);
  return (float)log(odds); /* log(float) promotes to double in C++ <cmath>? std::log(float) is the float overload */
}

/* GridMap(mapResolution, size, offset) with offset = mapSize*res*startCoords (MapRepMultiMap.h:63-67) */
orc_hmap *orc_hmap_create(int size_x, int size_y, float resolution, float start_x, float start_y) {
  orc_hmap *m = (orc_hmap *)calloc(1, sizeof(orc_hmap));
  m->size_x = size_x; m->size_y = size_y;
  float total_x = resolution * (float)size_x, total_y = resolution * (float)size_y;
  m->off_x = total_x * start_x;
  m->off_y = total_y * start_y;
  m->cell_length = resolution;
  m->scale_to_map = 1.0f / resolution;                      /* GridMapBase.h:276 */
  /* AlignedScaling2f(s,s) * Translation2f(off): linear diag(s,s), translation (s*offx, s*offy) */
  m->tw_lin = m->scale_to_map;
  m->tw_tx = m->scale_to_map * m->off_x;
  m->tw_ty = m->scale_to_map * m->off_y;
  /* Affine inverse: 2x2 cofactor inverse of diag(s,s), translation -(inv * t) */
  float det = m->tw_lin * m->tw_lin - 0.0f * 0.0f;
  float invdet = 1.0f / det;
  m->wt_lin = m->tw_lin * invdet;
  float i01 = -0.0f * invdet;
  m->wt_tx = -(m->wt_lin * m->tw_tx + i01 * m->tw_ty);
  m->wt_ty = -(i01 * m->tw_tx + m->wt_lin * m->tw_ty);
  m->log_odds_free = prob_to_log_odds(0.4f);                /* GridMapLogOdds.h:98-102 */
  m->log_odds_occ = prob_to_log_odds(0.6f);
  m->curr_update_index = 0;
  size_t n = (size_t)size_x * size_y;
  m->log_odds = (float *)calloc(n, sizeof(float));          /* resetGridCell: 0.0f, -1 (GridMapLogOdds.h:76-80) */
  m->update_index = (int32_t *)malloc(n * sizeof(int32_t));
  for (size_t i = 0; i < n; i++) m->update_index[i] = -1;
  return m;
}

void orc_hmap_destroy(orc_hmap *m) {
  if (!m) return;
  free(m->log_odds); free(m->update_index); free(m);
}

void orc_hmap_set_factors(orc_hmap *m, float update_free, float update_occ) {
  m->log_odds_free = prob_to_log_odds(update_free);
  m->log_odds_occ = prob_to_log_odds(update_occ);
}

void orc_hmap_copy(const orc_hmap *m, float *log_odds, int32_t *update_index) {
  size_t n = (size_t)m->size_x * m->size_y;
  if (log_odds) memcpy(log_odds, m->log_odds, n * sizeof(float));
  if (update_index) memcpy(update_index, m->update_index, n * sizeof(int32_t));
}

static void map_coords_pose(const orc_hmap *m, const float w[3], float out[3]) { /* GridMapBase.h:238-242 */
  out[0] = (m->tw_lin * w[0] + 0.0f * w[1]) + m->tw_tx;
  out[1] = (0.0f * w[0] + m->tw_lin * w[1]) + m->tw_ty;
  out[2] = w[2];
}
static void world_coords_pose(const orc_hmap *m, const float p[3], float out[3]) { /* GridMapBase.h:229-233 */
  out[0] = (m->wt_lin * p[0] + (-0.0f) * p[1]) + m->wt_tx; /* off-diagonal of the inverse is -0*invdet */
  out[1] = ((-0.0f) * p[0] + m->wt_lin * p[1]) + m->wt_ty;
  out[2] = p[2];
}

static void cell_free(orc_hmap *m, unsigned int off, int mark_free) { /* OccGridMapBase.h:302-312 */
  if (m->update_index[off] < mark_free) {
    m->log_odds[off] += m->log_odds_free;
    m->update_index[off] = mark_free;
  }
}
static void cell_occ(orc_hmap *m, unsigned int off, int mark_free, int mark_occ) { /* OccGridMapBase.h:315-330 */
  if (m->update_index[off] < mark_occ) {
    if (m->update_index[off] == mark_free) m->log_odds[off] -= m->log_odds_free;
    if (m->log_odds[off] < 50.0f) m->log_odds[off] += m->log_odds_occ;
    m->update_index[off] = mark_occ;
  }
}

static int hsign(int x) { return x > 0 ? 1 : -1; } /* util::sign (UtilFunctions.h:55-58): sign(0) = -1 */

/* updateLineBresenhami + bresenham2D (OccGridMapBase.h:220-299); returns cells touched (incl. end) */
static int update_line(orc_hmap *m, int x0, int y0, int x1, int y1, int mark_free, int mark_occ) {
  if (x0 < 0 || x0 >= m->size_x || y0 < 0 || y0 >= m->size_y) return 0;
  if (x1 < 0 || x1 >= m->size_x || y1 < 0 || y1 >= m->size_y) return 0;
  int dx = x1 - x0, dy = y1 - y0;
  unsigned int abs_dx = (unsigned int)abs(dx), abs_dy = (unsigned int)abs(dy);
  int offset_dx = hsign(dx), offset_dy = hsign(dy) * m->size_x;
  unsigned int offset = (unsigned int)(y0 * m->size_x + x0);
  unsigned int abs_da, abs_db;
  int error_b, offset_a, offset_b;
  if (abs_dx >= abs_dy) { abs_da = abs_dx; abs_db = abs_dy; error_b = (int)(abs_dx / 2); offset_a = offset_dx; offset_b = offset_dy; }
  else { abs_da = abs_dy; abs_db = abs_dx; error_b = (int)(abs_dy / 2); offset_a = offset_dy; offset_b = offset_dx; }
  int touched = 1;
  cell_free(m, offset, mark_free);
  unsigned int end = abs_da - 1;
  for (unsigned int i = 0; i < end; ++i) {
    offset += (unsigned int)offset_a;
    error_b += (int)abs_db;
    if ((unsigned int)error_b >= abs_da) {
      offset += (unsigned int)offset_b;
      error_b -= (int)abs_da;
    }
    cell_free(m, offset, mark_free);
    touched++;
  }
  cell_occ(m, (unsigned int)(y1 * m->size_x + x1), mark_free, mark_occ);
  return touched + 1;
}

/* OccGridMapBase::updateByScan (OccGridMapBase.h:118-168).  points = DataContainer entries (map-cell units),
 * origo likewise, world_pose = robot pose in world coordinates.  Returns the number of cell visits. */
long orc_hmap_update_by_scan(orc_hmap *m, const float *points, int n, const float origo[2], const float world_pose[3]) {
  int mark_free = m->curr_update_index + 1, mark_occ = m->curr_update_index + 2;
  float mp[3];
  map_coords_pose(m, world_pose, mp);
  float c = cosf(mp[2]), s = sinf(mp[2]); /* Eigen::Rotation2Df(angle).toRotationMatrix(): std::cos/std::sin(float) */
  float bx = (c * origo[0] + (-s) * origo[1]) + mp[0];
  float by = (s * origo[0] + c * origo[1]) + mp[1];
  int bxi = (int)(bx + 0.5f), byi = (int)(by + 0.5f);
  long visits = 0;
  for (int i = 0; i < n; i++) {
    float ex = (c * points[2 * i] + (-s) * points[2 * i + 1]) + mp[0];
    float ey = (s * points[2 * i] + c * points[2 * i + 1]) + mp[1];
    ex += 0.5f; ey += 0.5f;
    int exi = (int)ex, eyi = (int)ey;
    if (bxi != exi || byi != eyi) visits += update_line(m, bxi, byi, exi, eyi, mark_free, mark_occ);
  }
  m->curr_update_index += 3;
  return visits;
}

/* getGridProbability (GridMapLogOdds.h:136-140) */
/* OccGridMapBase::updateByScanJustOnce (OccGridMapBase.h:175-217), the lesson4 make-map demo variant: fixed map
 * pose (800, 800, 0); points are in METRES and the end cell is begin + (int)round(p / 0.05) in double. */
long orc_hmap_update_by_scan_just_once(orc_hmap *m, const float *points, int n, const float origo[2]) {
  int mark_free = m->curr_update_index + 1, mark_occ = m->curr_update_index + 2;
  float mp[3] = {800.0f, 800.0f, 0.0f};
  float c = cosf(mp[2]), s = sinf(mp[2]);
  float bx = (c * origo[0] + (-s) * origo[1]) + mp[0];
  float by = (s * origo[0] + c * origo[1]) + mp[1];
  int bxi = (int)(bx + 0.5f), byi = (int)(by + 0.5f);
  long visits = 0;
  for (int i = 0; i < n; i++) {
    int exi = bxi + (int)round(points[2 * i] / 0.05);
    int eyi = byi + (int)round(points[2 * i + 1] / 0.05);
    if (bxi != exi || byi != eyi) visits += update_line(m, bxi, byi, exi, eyi, mark_free, mark_occ);
  }
  m->curr_update_index += 3;
  return visits;
}

/* getGridProbability (GridMapLogOdds.h:136-140): `float odds = exp(cell.logOddsVal);` — the header includes only
 * <cmath>, so the unqualified exp / sin / cos on a float resolve to the C library's DOUBLE functions (the reference
 * build imports exp, sincos, sincosf, log, fmod, pow, round and no expf: `nm -D oracle/_ref/libhector_ref.so`); the
 * result is rounded to float on assignment.  (float)exp((double)x) and expf(x) differ on ~0.07 % of inputs. */
static float grid_prob(const orc_hmap *m, int index) {
  float odds = (float)exp((double)m->log_odds[index]);
  return odds / (odds + 1.0f);
}

void orc_hector_grid_probabilities(const float *log_odds, int n, float *out) {
  orc_hmap m;
  memset(&m, 0, sizeof(m));
  m.log_odds = (float *)log_odds;
  for (int i = 0; i < n; i++) out[i] = grid_prob(&m, i);
}

/* interpMapValueWithDerivatives (OccGridMapUtil.h:139-228); the per-scan cache only memoises getGridProbability */
static void interp(const orc_hmap *m, float x, float y, float out[3]) {
  float lim_x = (float)m->size_x - 2.0f, lim_y = (float)m->size_y - 2.0f; /* setMapCellDims: dims - 2 */
  if (x < 0.0f || x > lim_x || y < 0.0f || y > lim_y) { out[0] = out[1] = out[2] = 0.0f; return; }
  /* A NaN coordinate (a pose that went through a singular Hessian) passes the test above.  The reference's (int) of
   * NaN is undefined (x86 gives INT_MIN and reads far outside the map); here it is 0, as the device's conversion
   * (cvt.rzi.s32.f32) gives, so the read stays inside and the NaN reaches the outputs through fx / fy. */
  int ix = x == x ? (int)x : 0, iy = y == y ? (int)y : 0;
  float fx = x - (float)ix, fy = y - (float)iy;
  int index = iy * m->size_x + ix;
  float i0 = grid_prob(m, index), i1 = grid_prob(m, index + 1);
  float i2 = grid_prob(m, index + m->size_x), i3 = grid_prob(m, index + m->size_x + 1);
  float dx1 = i0 - i1, dx2 = i2 - i3, dy1 = i0 - i2, dy2 = i1 - i3;
  float xfi = 1.0f - fx, yfi = 1.0f - fy;
  out[0] = ((i0 * xfi + i1 * fx) * yfi) + ((i2 * xfi + i3 * fx) * fy);
  out[1] = -((dx1 * yfi) + (dx2 * fy));
  out[2] = -((dy1 * xfi) + (dy2 * fx));
}

/* getCompleteHessianDerivs (OccGridMapUtil.h:77-132): H row-major 3x3, dTr[3] */
static void hessian_derivs(const orc_hmap *m, const float pose[3], const float *pts, int n, float H[9], float dTr[3]) {
  float c = cosf(pose[2]), s = sinf(pose[2]);          /* getTransformForState: Rotation2Df */
  float sin_rot = (float)sin((double)pose[2]), cos_rot = (float)cos((double)pose[2]); /* unqualified sin / cos: ::sin(double), rounded to float */
  memset(H, 0, 9 * sizeof(float));
  memset(dTr, 0, 3 * sizeof(float));
  for (int i = 0; i < n; i++) {
    float px = pts[2 * i], py = pts[2 * i + 1];
    float tx = (c * px + (-s) * py) + pose[0], ty = (s * px + c * py) + pose[1];
    float t[3];
    interp(m, tx, ty, t);
    float fun = 1.0f - t[0];
    dTr[0] += t[1] * fun;
    dTr[1] += t[2] * fun;
    float rot = ((-sin_rot * px - cos_rot * py) * t[1] + (cos_rot * px - sin_rot * py) * t[2]);
    dTr[2] += rot * fun;
    H[0] += t[1] * t[1];
    H[4] += t[2] * t[2];
    H[8] += rot * rot;
    H[1] += t[1] * t[2];
    H[2] += t[1] * rot;
    H[5] += t[2] * rot;
  }
  H[3] = H[1]; H[6] = H[2]; H[7] = H[5];
}

static float hnormalize_angle(float angle) { /* UtilFunctions.h:36-48 (double fmod, float return) */
  float a = (float)fmod(fmod((double)angle, 2.0f * M_PI) + 2.0f * M_PI, 2.0f * M_PI);
  if (a > M_PI) a = (float)((double)a - 2.0f * M_PI); /* `a -= 2.0f*M_PI` is evaluated in double */
  return a;
}

/* Matrix3f::inverse() * v, cofactor / determinant form (Eigen compute_inverse_size3) */
static void inv3_mul(const float m[9], const float v[3], float out[3]) {
  float c00 = m[4] * m[8] - m[5] * m[7], c10 = m[5] * m[6] - m[3] * m[8], c20 = m[3] * m[7] - m[4] * m[6];
  float det = c00 * m[0] + (c10 * m[1] + c20 * m[2]);  /* Eigen's unrolled 3-term redux: a0 + (a1 + a2) */
  float invdet = 1.0f / det;
  float inv[9];
  inv[0] = c00 * invdet; inv[3] = c10 * invdet; inv[6] = c20 * invdet;
  inv[1] = (m[2] * m[7] - m[1] * m[8]) * invdet;
  inv[4] = (m[0] * m[8] - m[2] * m[6]) * invdet;
  inv[7] = (m[1] * m[6] - m[0] * m[7]) * invdet;
  inv[2] = (m[1] * m[5] - m[2] * m[4]) * invdet;
  inv[5] = (m[2] * m[3] - m[0] * m[5]) * invdet;
  inv[8] = (m[0] * m[4] - m[1] * m[3]) * invdet;
  for (int r = 0; r < 3; r++) out[r] = inv[3 * r] * v[0] + (inv[3 * r + 1] * v[1] + inv[3 * r + 2] * v[2]);
}

/* ScanMatcher::matchData (ScanMatcher.h:60-98): 1 + max_iterations Gauss-Newton steps on one grid level */
void orc_hmap_match_data(const orc_hmap *m, const float *pts, int n, const float begin_world[3], int max_iterations,
                         float out_world[3], float out_cov[9]) {
  if (n == 0) {
    memcpy(out_world, begin_world, 3 * sizeof(float));
    return;
  }
  float est[3], H[9], dTr[3];
  map_coords_pose(m, begin_world, est);
  for (int it = 0; it < 1 + max_iterations; it++) { /* estimateTransformationLogLh (ScanMatcher.h:107-141) */
    hessian_derivs(m, est, pts, n, H, dTr);
    if (H[0] != 0.0f && H[4] != 0.0f) {
      float dir[3];
      inv3_mul(H, dTr, dir);
      if (dir[2] > 0.2f) dir[2] = 0.2f;
      else if (dir[2] < -0.2f) dir[2] = -0.2f;
      est[0] += dir[0]; est[1] += dir[1]; est[2] += dir[2];
    }
  }
  est[2] = hnormalize_angle(est[2]);
  memcpy(out_cov, H, 9 * sizeof(float));
  world_coords_pose(m, est, out_world);
}

/* ------------------------------------------------------------------------------------------------------------
 * HectorSlamProcessor (slam_main/HectorSlamProcessor.h:53-125) over MapRepMultiMap (slam_main/MapRepMultiMap.h:56-191):
 * the lesson4 front end.  PINNED against the reference headers compiled with the Eigen stand-in
 * (oracle/ref_hector.cpp, tests/test_oracle_hector_reference.py).
 * ------------------------------------------------------------------------------------------------------------ */
#define ORC_HPROC_MAX_LEVELS 8
typedef struct {
  int levels;
  orc_hmap *map[ORC_HPROC_MAX_LEVELS];
  float *pts[ORC_HPROC_MAX_LEVELS];   /* dataContainers[level-1]: the last MATCHED scan scaled by 1/2^level */
  int n_pts[ORC_HPROC_MAX_LEVELS];
  float origo[ORC_HPROC_MAX_LEVELS][2];
  float last_map_update_pose[3], last_scan_match_pose[3], last_cov[9];
  float min_dist, min_angle;
  int map_updated; /* the last update()'s gate decision (the device handle reports it per scan) */
} orc_hproc;

orc_hproc *orc_hproc_create(float resolution, int size_x, int size_y, float start_x, float start_y, int levels) {
  if (levels < 1 || levels > ORC_HPROC_MAX_LEVELS) return NULL;
  orc_hproc *p = (orc_hproc *)calloc(1, sizeof(orc_hproc));
  p->levels = levels;
  /* MapRepMultiMap.h:61-86: ONE offset (level-0 size * resolution * startCoords) for every level; dims halve by
   * integer division, the cell length doubles */
  float total_x = resolution * (float)size_x, total_y = resolution * (float)size_y;
  float off_x = total_x * start_x, off_y = total_y * start_y;
  for (int l = 0; l < levels; l++) {
    orc_hmap *m = orc_hmap_create(size_x, size_y, resolution, 0.0f, 0.0f);
    m->off_x = off_x; m->off_y = off_y;
    m->tw_tx = m->scale_to_map * off_x; m->tw_ty = m->scale_to_map * off_y;
    float det = m->tw_lin * m->tw_lin - 0.0f * 0.0f, invdet = 1.0f / det, i01 = -0.0f * invdet;
    m->wt_tx = -(m->wt_lin * m->tw_tx + i01 * m->tw_ty);
    m->wt_ty = -(i01 * m->tw_tx + m->wt_lin * m->tw_ty);
    p->map[l] = m;
    size_x /= 2; size_y /= 2;
    resolution *= 2.0f;
  }
  /* reset() (HectorSlamProcessor.h:111-116); ctor thresholds (:63-64) */
  p->last_map_update_pose[0] = p->last_map_update_pose[1] = p->last_map_update_pose[2] = 3.402823466e+38F;
  p->min_dist = 0.4f * 1.0f;
  p->min_angle = 0.13f * 1.0f;
  return p;
}

void orc_hproc_destroy(orc_hproc *p) {
  if (!p) return;
  for (int l = 0; l < p->levels; l++) { orc_hmap_destroy(p->map[l]); free(p->pts[l]); }
  free(p);
}

void orc_hproc_set_params(orc_hproc *p, float update_free, float update_occ, float min_dist, float min_angle) {
  for (int l = 0; l < p->levels; l++) orc_hmap_set_factors(p->map[l], update_free, update_occ);
  p->min_dist = min_dist;
  p->min_angle = min_angle;
}

/* util::poseDifferenceLargerThan (UtilFunctions.h:72-90).  The header includes only <cmath>, so the unqualified
 * `abs(angleDiff)` resolves to `int abs(int)`: the angle difference is TRUNCATED to an integer before the compare
 * (verified on the reference build: a 0.5 rad turn with angleDiffThresh 0.13 returns false). */
static int pose_difference_larger_than(const float a[3], const float b[3], float dist_thresh, float angle_thresh) {
  float dx = a[0] - b[0], dy = a[1] - b[1];
  if (sqrtf(dx * dx + dy * dy) > dist_thresh) return 1;
  float d = a[2] - b[2];
  if (d > M_PI) d = (float)((double)d - M_PI * 2.0f);
  else if (d < -M_PI) d = (float)((double)d + M_PI * 2.0f);
  return (float)abs((int)d) > angle_thresh;
}

/* DataPointContainer::setFrom (DataPointContainer.h:46-59) */
static void set_from(orc_hproc *p, int l, const float *points, int n, const float origo[2], float factor) {
  p->pts[l] = (float *)realloc(p->pts[l], (size_t)(n > 0 ? n : 1) * 2 * sizeof(float));
  p->n_pts[l] = n;
  p->origo[l][0] = origo[0] * factor; p->origo[l][1] = origo[1] * factor;
  for (int i = 0; i < 2 * n; i++) p->pts[l][i] = points[i] * factor;
}

/* HectorSlamProcessor::update (:81-108).  points/origo in level-0 map-cell units; pose hint in world metres. */
void orc_hproc_update(orc_hproc *p, const float *points, int n, const float origo[2], const float pose_hint[3],
                      int map_without_matching, float out_pose[3], float out_cov[9]) {
  float est[3];
  if (!map_without_matching) { /* MapRepMultiMap::matchData (:144-166): coarsest level first */
    float tmp[3] = {pose_hint[0], pose_hint[1], pose_hint[2]};
    for (int l = p->levels - 1; l >= 0; l--) {
      float next[3];
      if (l == 0) {
        orc_hmap_match_data(p->map[0], points, n, tmp, 5, next, p->last_cov);
      } else {
        set_from(p, l, points, n, origo, (float)(1.0 / pow(2.0, (double)l)));
        orc_hmap_match_data(p->map[l], p->pts[l], n, tmp, 3, next, p->last_cov);
      }
      memcpy(tmp, next, sizeof(tmp));
    }
    memcpy(est, tmp, sizeof(est));
  } else {
    memcpy(est, pose_hint, sizeof(est));
  }
  memcpy(p->last_scan_match_pose, est, sizeof(est));
  p->map_updated = pose_difference_larger_than(est, p->last_map_update_pose, p->min_dist, p->min_angle) || map_without_matching;
  if (p->map_updated) {
    /* MapRepMultiMap::updateByScan (:174-191): the coarse levels use dataContainers filled by the LAST matchData —
     * with map_without_matching they are stale (empty before the first match); reproduced as is */
    for (int l = 0; l < p->levels; l++) {
      if (l == 0) orc_hmap_update_by_scan(p->map[0], points, n, origo, est);
      else orc_hmap_update_by_scan(p->map[l], p->pts[l], p->n_pts[l], p->origo[l], est);
    }
    memcpy(p->last_map_update_pose, est, sizeof(est));
  }
  memcpy(out_pose, est, sizeof(est));
  if (out_cov && !map_without_matching) memcpy(out_cov, p->last_cov, sizeof(p->last_cov));
}

int orc_hproc_map_updated(const orc_hproc *p) { return p->map_updated; }

int orc_hproc_level_dims(const orc_hproc *p, int level, int dims[2]) {
  if (level < 0 || level >= p->levels) return -1;
  dims[0] = p->map[level]->size_x; dims[1] = p->map[level]->size_y;
  return 0;
}

void orc_hproc_copy_level(const orc_hproc *p, int level, float *log_odds, int32_t *update_index) {
  orc_hmap_copy(p->map[level], log_odds, update_index);
}
