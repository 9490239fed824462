/*
 * karto_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C, single-threaded CPU restatement of the reference's Karto hot path
 * (K1 correlative scan matcher + K2c occupancy grid), function by function, each citing
 * the reference file:line it follows (paths relative to reference/lesson6/lib/open_karto).
 * It exists so the CUDA path can be checked on the GPU box, where the reference checkout is absent.
 *
 * PARITY PINNED: tests/test_oracle_vs_reference.py checks every function here against the
 * UNMODIFIED reference compiled by oracle/recipes.py (oracle/_ref/libkarto_ref.so), bit-exact
 * on grid bytes / lookup tables / integer response sums / counters and to 1e-12 on doubles, and
 * tests/golden/ holds vectors produced by that reference build (tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  The product (libb200slam.so) never links or calls it.
 *
 * Build: gcc -O2 -ffp-contract=off (no FMA contraction: the reference's x86-64 build has none).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h" /* struct layouts only */
#include "oracle_common.h"

#define KT_PI 3.14159265358979323846  /* include/open_karto/Math.h:32 */
#define KT_2PI 6.28318530717958647692 /* Math.h:33 */
#define KT_TOLERANCE 1e-06            /* Math.h:41 */
#define INVALID_SCAN INT32_MAX        /* Math.h:47 */
#define GRID_OCCUPIED 100             /* Karto.h:4196 */
#define GRID_FREE 255                 /* Karto.h:4197 */
#define MAX_VARIANCE 500.0            /* src/Mapper.cpp:36 */
#define DISTANCE_PENALTY_GAIN 0.2     /* Mapper.cpp:37 */
#define ANGLE_PENALTY_GAIN 0.2        /* Mapper.cpp:38 */

/* math::Round (Math.h:87-90): half away from zero */
double orc_round(double v) { return v >= 0.0 ? floor(v + 0.5) : ceil(v - 0.5); }

/* math::DoubleEqual (Math.h:135-139) */
static int double_equal(double a, double b) {
  double delta = a - b;
  return delta < 0.0 ? delta >= -KT_TOLERANCE : delta <= KT_TOLERANCE;
}

/* math::NormalizeAngle (Math.h:182-211) */
double orc_normalize_angle(double angle) {
  while (angle < -KT_PI) {
    if (angle < -KT_2PI)
      angle += (uint32_t)(angle / -KT_2PI) * KT_2PI;
    else
      angle += KT_2PI;
  }
  while (angle > KT_PI) {
    if (angle > KT_2PI)
      angle -= (uint32_t)(angle / KT_2PI) * KT_2PI;
    else
      angle -= KT_2PI;
  }
  return angle;
}

/* math::NormalizeAngleDifference (Math.h:221-234) */
static double normalize_angle_difference(double minuend, double subtrahend) {
  while (minuend - subtrahend < -KT_PI) minuend += KT_2PI;
  while (minuend - subtrahend > KT_PI) minuend -= KT_2PI;
  return minuend;
}

static double dmax(double a, double b) { return a > b ? a : b; } /* math::Maximum (Math.h:110-114) */

/* CoordinateConverter::WorldToGrid, one axis (Karto.h:4237-4252) */
static int32_t world_to_grid_1(double w, double offset, double scale) {
  return (int32_t)orc_round((w - offset) * scale);
}

/* ScanMatcher::Create sizing (Mapper.cpp:126-172) + CorrelationGrid::CreateGrid / ctor (Mapper.h:920-1027)
 * + Grid::Resize width step (Karto.h:4438-4442) + CalculateKernel range check (Mapper.h:1039-1053). */
int orc_matcher_layout(const b2s_matcher_params *p, b2s_grid_info *g) {
  if (p->resolution <= 0) return B2S_ERR_BAD_PARAMS;
  if (p->search_size <= 0) return B2S_ERR_BAD_PARAMS;
  if (p->smear_deviation < 0) return B2S_ERR_BAD_PARAMS;
  if (p->range_threshold <= 0) return B2S_ERR_BAD_PARAMS;
  uint32_t side = (uint32_t)(orc_round(p->search_size / p->resolution) + 1);
  uint32_t margin = (uint32_t)ceil(p->range_threshold / p->resolution);
  int32_t grid_size = (int32_t)(side + 2 * margin);
  int32_t half_kernel = (int32_t)orc_round(2.0 * p->smear_deviation / p->resolution); /* Mapper.h:1096-1101 */
  uint32_t border = (uint32_t)(half_kernel + 1);                                     /* Mapper.h:928 */
  g->width = grid_size + 2 * (int32_t)border;
  g->height = grid_size + 2 * (int32_t)border;
  g->width_step = (int32_t)(((size_t)g->width + 7) & ~(size_t)7); /* Math.h:243-247 */
  g->data_size = g->width_step * g->height;
  g->roi_x = g->roi_y = (int32_t)border;
  g->roi_w = g->roi_h = grid_size;
  g->kernel_size = 2 * half_kernel + 1;
  g->search_side = (int32_t)side;
  /* CalculateKernel: resolution read back as 1/(1/res) (Mapper.h:1020,1034; Karto.h:4335-4338) */
  double resolution = 1.0 / (1.0 / p->resolution);
  double min_dev = 0.5 * resolution, max_dev = 10 * resolution;
  if (!(p->smear_deviation >= min_dev && p->smear_deviation <= max_dev)) return B2S_ERR_BAD_PARAMS;
  return B2S_OK;
}

/* CorrelationGrid::CalculateKernel (Mapper.h:1032-1087): K[(i+h) + ksize*(j+h)] */
void orc_smear_kernel(double resolution_param, double smear, int ksize, uint8_t *K) {
  double resolution = 1.0 / (1.0 / resolution_param);
  int half = ksize / 2;
  for (int i = -half; i <= half; i++)
    for (int j = -half; j <= half; j++) {
      double d = hypot(i * resolution, j * resolution);
      double z = exp(-0.5 * pow(d / smear, 2));
      uint32_t kv = (uint32_t)orc_round(z * GRID_OCCUPIED);
      K[(i + half) + ksize * (j + half)] = (uint8_t)kv;
    }
}

/* LocalizedRangeScan::GetSensorAt = Transform(robotPose).TransformPose(offsetPose)
 * (Karto.h:5310-5313, 2860-2887, 2909-2935; Matrix3::FromAxisAngle 2392-2421; Matrix3*Pose2 2574-2583) */
void orc_sensor_pose(const double robot[3], const double offset[3], double out[3]) {
  double m00, m01, m02, m10, m11, m12, tx, ty, th;
  if (robot[0] == 0.0 && robot[1] == 0.0 && robot[2] == 0.0) { /* rPose1 == rPose2 (Karto.h:2911-2917) */
    m00 = 1; m01 = 0; m02 = 0; m10 = 0; m11 = 1; m12 = 0; tx = 0; ty = 0; th = 0;
  } else {
    double radians = robot[2] - 0.0;
    double c = cos(radians), s = sin(radians), omc = 1.0 - c;
    /* axis (0,0,1): xx=yy=0, zz=1, every mixed term is 0*omc or 0*s */
    m00 = 0.0 * omc + c;
    m01 = 0.0 * 0.0 * omc - 1.0 * s;
    m02 = 0.0 * 1.0 * omc + 0.0 * s;
    m10 = 0.0 * 0.0 * omc + 1.0 * s;
    m11 = 0.0 * omc + c;
    m12 = 0.0 * 1.0 * omc - 0.0 * s;
    tx = robot[0]; ty = robot[1]; th = robot[2] - 0.0;
  }
  double rx = m00 * offset[0] + m01 * offset[1] + m02 * offset[2];
  double ry = m10 * offset[0] + m11 * offset[1] + m12 * offset[2];
  out[0] = tx + rx;
  out[1] = ty + ry;
  out[2] = orc_normalize_angle(offset[2] + th);
}

/* LocalizedRangeScan::Update, unfiltered list (Karto.h:5362-5404): every reading yields a point */
void orc_point_readings(const b2s_laser *l, const double *ranges, const double robot_pose[3], double *out_xy) {
  double sp[3];
  orc_sensor_pose(robot_pose, l->offset_pose, sp);
  for (int i = 0; i < l->n_readings; i++) {
    double angle = sp[2] + l->min_angle + (uint32_t)i * l->angular_resolution;
    out_xy[2 * i] = sp[0] + (ranges[i] * cos(angle));
    out_xy[2 * i + 1] = sp[1] + (ranges[i] * sin(angle));
  }
}

/* filtered list + bounding box (Karto.h:5382,5400,5418-5424): bbox over sensor position and points whose
 * reading is InRange(minRange, rangeThreshold).  bbox = {minx, miny, maxx, maxy}. */
void orc_scan_bbox(const b2s_laser *l, const double *ranges, const double robot_pose[3], double bbox[4]) {
  double sp[3];
  orc_sensor_pose(robot_pose, l->offset_pose, sp);
  double mnx = 999999999999999999.99999, mny = mnx, mxx = -mnx, mxy = -mnx; /* Karto.h:2765 */
  if (sp[0] < mnx) mnx = sp[0];
  if (sp[1] < mny) mny = sp[1];
  if (sp[0] > mxx) mxx = sp[0];
  if (sp[1] > mxy) mxy = sp[1];
  for (int i = 0; i < l->n_readings; i++) {
    double r = ranges[i];
    if (!(r >= l->min_range && r <= l->range_threshold)) continue;
    double angle = sp[2] + l->min_angle + (uint32_t)i * l->angular_resolution;
    double x = sp[0] + (r * cos(angle)), y = sp[1] + (r * sin(angle));
    if (x < mnx) mnx = x;
    if (y < mny) mny = y;
    if (x > mxx) mxx = x;
    if (y > mxy) mxy = y;
  }
  bbox[0] = mnx; bbox[1] = mny; bbox[2] = mxx; bbox[3] = mxy;
}

/* ScanMatcher::FindValidPoints (Mapper.cpp:756-811).  Returns the number of points written. */
int orc_find_valid_points(const double *pts_xy, int n, const double viewpoint[2], double *out_xy) {
  const double min_sq = 0.1 * 0.1;
  int trailing = 0, n_out = 0;
  double fx = 0.0, fy = 0.0; /* Vector2<kt_double> firstPoint default = (0,0) */
  int first_time = 1;
  for (int it = 0; it < n; it++) {
    double cx = pts_xy[2 * it], cy = pts_xy[2 * it + 1];
    if (first_time && !isnan(cx) && !isnan(cy)) {
      fx = cx; fy = cy;
      first_time = 0;
    }
    double dx = fx - cx, dy = fy - cy;
    if (dx * dx + dy * dy > min_sq) {
      double a = viewpoint[1] - fy;
      double b = fx - viewpoint[0];
      double c = fy * viewpoint[0] - fx * viewpoint[1];
      double ss = cx * a + cy * b + c;
      fx = cx; fy = cy;
      if (ss < 0.0) {
        trailing = it;
      } else {
        for (; trailing != it; ++trailing) {
          out_xy[2 * n_out] = pts_xy[2 * trailing];
          out_xy[2 * n_out + 1] = pts_xy[2 * trailing + 1];
          n_out++;
        }
      }
    }
  }
  return n_out;
}

/* MatchScan steps 2-4 (Mapper.cpp:212-220): grid offset so that the ROI centre is the scan's sensor position */
void orc_grid_offset(const b2s_grid_info *g, double resolution_param, const double sensor_pose[3], double off[2]) {
  double resolution = 1.0 / (1.0 / resolution_param); /* GetResolution() = 1/scale, scale = 1/res */
  off[0] = sensor_pose[0] - (0.5 * (g->roi_w - 1) * resolution);
  off[1] = sensor_pose[1] - (0.5 * (g->roi_h - 1) * resolution);
}

/* CorrelationGrid::SmearPoint (Mapper.h:971-1005); gx, gy are ROI-relative */
static void smear_point(const b2s_grid_info *g, uint8_t *grid, const uint8_t *K, int gx, int gy) {
  int half = g->kernel_size / 2;
  for (int j = -half; j <= half; j++) {
    uint8_t *adr = grid + (gx + g->roi_x) + (gy + j + g->roi_y) * g->width_step;
    int kc = half + g->kernel_size * (j + half);
    for (int i = -half; i <= half; i++) {
      uint8_t kv = K[i + kc];
      if (kv > adr[i]) adr[i] = kv;
    }
  }
}

/* ScanMatcher::AddScan for ONE base scan given its unfiltered point readings (Mapper.cpp:716-748) */
void orc_add_scan(const b2s_grid_info *g, double resolution_param, const double grid_off[2], uint8_t *grid,
                  const uint8_t *K, const double *pts_xy, int n, const double viewpoint[2], double *scratch_xy) {
  double scale = 1.0 / resolution_param; /* CorrelationGrid ctor SetScale (Mapper.h:1020) */
  int nv = orc_find_valid_points(pts_xy, n, viewpoint, scratch_xy);
  for (int i = 0; i < nv; i++) {
    double gxd = orc_round((scratch_xy[2 * i] - grid_off[0]) * scale);
    double gyd = orc_round((scratch_xy[2 * i + 1] - grid_off[1]) * scale);
    /* static_cast<kt_int32s> of a non-finite / huge double is UB in the reference (x86: INT_MIN, rejected
     * by IsUpTo).  Restated as an explicit reject. */
    if (!(gxd >= 0.0 && gxd < (double)g->roi_w) || !(gyd >= 0.0 && gyd < (double)g->roi_h)) continue;
    int gx = (int)gxd, gy = (int)gyd;
    int idx = (gx + g->roi_x) + (gy + g->roi_y) * g->width_step;
    if (grid[idx] == GRID_OCCUPIED) continue;
    grid[idx] = GRID_OCCUPIED;
    smear_point(g, grid, K, gx, gy);
  }
}

/* ScanMatcher::AddScans (Mapper.cpp:699-708) over n_base scans given as ranges + robot poses.
 * viewpoint = scanPose.GetPosition() of the scan being matched (Mapper.cpp:225). */
void orc_add_scans(const b2s_matcher_params *p, const b2s_laser *l, const b2s_grid_info *g, const double grid_off[2],
                   uint8_t *grid, int n_base, const double *base_ranges, const double *base_poses,
                   const double viewpoint[2]) {
  int n = l->n_readings;
  uint8_t *K = (uint8_t *)malloc((size_t)g->kernel_size * g->kernel_size);
  double *pts = (double *)malloc(sizeof(double) * 2 * (size_t)n);
  double *scratch = (double *)malloc(sizeof(double) * 2 * (size_t)n);
  orc_smear_kernel(p->resolution, p->smear_deviation, g->kernel_size, K);
  memset(grid, 0, (size_t)g->data_size); /* Grid::Clear (Karto.h:4414-4417) */
  for (int s = 0; s < n_base; s++) {
    orc_point_readings(l, base_ranges + (size_t)s * n, base_poses + 3 * (size_t)s, pts);
    orc_add_scan(g, p->resolution, grid_off, grid, K, pts, n, viewpoint, scratch);
  }
  free(K); free(pts); free(scratch);
}

/* number of search steps: static_cast<kt_int32u>(math::Round(off * 2.0 / res) + 1) (Mapper.cpp:339-341,361) */
int orc_n_steps(double off, double res) { return (int)(uint32_t)(orc_round(off * 2.0 / res) + 1); }

/* GridIndexLookup::ComputeOffsets (Karto.h:6409-6501).  pts_xy = the scan's unfiltered point readings,
 * sensor_pose = pScan->GetSensorPose().  lut[k*n + i]. */
void orc_compute_offsets(const b2s_grid_info *g, double resolution_param, const double grid_off[2],
                         const double *ranges, const double *pts_xy, int n, const double sensor_pose[3],
                         double angle_center, double angle_offset, double angle_res, int32_t *lut) {
  double scale = 1.0 / resolution_param;
  int n_angles = orc_n_steps(angle_offset, angle_res);
  double *lx = (double *)malloc(sizeof(double) * (size_t)n), *ly = (double *)malloc(sizeof(double) * (size_t)n);
  /* Transform(sensorPose).InverseTransformPose(Pose2(pt, 0)) (Karto.h:2894-2901, 2909-2935) */
  double i00, i01, i02, i10, i11, i12, tx, ty, th;
  if (sensor_pose[0] == 0.0 && sensor_pose[1] == 0.0 && sensor_pose[2] == 0.0) {
    i00 = 1; i01 = 0; i02 = 0; i10 = 0; i11 = 1; i12 = 0; tx = ty = th = 0;
  } else {
    double radians = 0.0 - sensor_pose[2];
    double c = cos(radians), s = sin(radians), omc = 1.0 - c;
    i00 = 0.0 * omc + c;
    i01 = 0.0 * 0.0 * omc - 1.0 * s;
    i02 = 0.0 * 1.0 * omc + 0.0 * s;
    i10 = 0.0 * 0.0 * omc + 1.0 * s;
    i11 = 0.0 * omc + c;
    i12 = 0.0 * 1.0 * omc - 0.0 * s;
    tx = sensor_pose[0]; ty = sensor_pose[1]; th = sensor_pose[2] - 0.0;
  }
  for (int i = 0; i < n; i++) {
    double dx = pts_xy[2 * i] - tx, dy = pts_xy[2 * i + 1] - ty;
    double dh = orc_normalize_angle(0.0 - th); /* Pose2::operator- heading (Karto.h:2138-2141) */
    lx[i] = i00 * dx + i01 * dy + i02 * dh;
    ly[i] = i10 * dx + i11 * dy + i12 * dh;
  }
  double start = angle_center - angle_offset;
  for (int k = 0; k < n_angles; k++) {
    double angle = start + (uint32_t)k * angle_res;
    double cosine = cos(angle), sine = sin(angle);
    for (int i = 0; i < n; i++) {
      if (isnan(ranges[i]) || isinf(ranges[i])) {
        lut[(size_t)k * n + i] = INVALID_SCAN;
        continue;
      }
      double ox = cosine * lx[i] - sine * ly[i];
      double oy = sine * lx[i] + cosine * ly[i];
      /* WorldToGrid(offset + rGridOffset): ((o + off) - off) * scale (Karto.h:6491, 4239-4251) */
      int32_t gx = (int32_t)orc_round(((ox + grid_off[0]) - grid_off[0]) * scale);
      int32_t gy = (int32_t)orc_round(((oy + grid_off[1]) - grid_off[1]) * scale);
      lut[(size_t)k * n + i] = gx + gy * g->width_step; /* Grid<T>::GridIndex, no ROI (Karto.h:4501,6494) */
    }
  }
  free(lx); free(ly);
}

/* integer numerator of ScanMatcher::GetResponse (Mapper.cpp:819-856) */
static int32_t response_sum(const uint8_t *grid, int32_t data_size, int32_t base, const int32_t *offs, int n) {
  int32_t sum = 0;
  for (int i = 0; i < n; i++) {
    if (offs[i] == INVALID_SCAN) continue; /* tested first: base + INT32_MAX is signed overflow in the reference */
    int32_t idx = base + offs[i];
    if (!(idx >= 0 && idx < data_size)) continue;
    sum += grid[idx];
  }
  return sum;
}

typedef struct {
  int nx, ny, na;
  int32_t *base; /* [ny*nx] flat grid index of each candidate position incl. ROI */
} sweep_layout;

/* candidate lattice of CorrelateScan (Mapper.cpp:338-358, 373-386); returns status */
static int sweep_bases(const b2s_grid_info *g, double resolution_param, const double grid_off[2],
                       const double center[3], const b2s_search *s, sweep_layout *L) {
  double scale = 1.0 / resolution_param;
  L->nx = orc_n_steps(s->offset_x, s->res_x);
  L->ny = orc_n_steps(s->offset_y, s->res_y);
  L->na = orc_n_steps(s->angle_offset, s->angle_res);
  L->base = (int32_t *)malloc(sizeof(int32_t) * (size_t)L->nx * L->ny);
  double start_x = -s->offset_x, start_y = -s->offset_y;
  for (int iy = 0; iy < L->ny; iy++) {
    double y = start_y + (uint32_t)iy * s->res_y;
    double new_y = center[1] + y;
    for (int ix = 0; ix < L->nx; ix++) {
      double x = start_x + (uint32_t)ix * s->res_x;
      double new_x = center[0] + x;
      int32_t gx = world_to_grid_1(new_x, grid_off[0], scale) + g->roi_x; /* CorrelationGrid::GridIndex */
      int32_t gy = world_to_grid_1(new_y, grid_off[1], scale) + g->roi_y; /* (Mapper.h:941-947)        */
      if (!(gx >= 0 && gx < g->width && gy >= 0 && gy < g->height)) { /* Karto.h:4490-4499 throws */
        free(L->base);
        L->base = NULL;
        return B2S_ERR_OUT_OF_RANGE;
      }
      L->base[iy * L->nx + ix] = gx + gy * g->width_step;
    }
  }
  return B2S_OK;
}

/* The response sweep of CorrelateScan as integer sums, out[ny][nx][na] (Mapper.cpp:373-424). */
int orc_response_sums(const b2s_grid_info *g, double resolution_param, const double grid_off[2], const uint8_t *grid,
                      const int32_t *lut, int n, const double center[3], const b2s_search *s, int32_t *out) {
  sweep_layout L;
  int rc = sweep_bases(g, resolution_param, grid_off, center, s, &L);
  if (rc) return rc;
  size_t w = 0;
  for (int iy = 0; iy < L.ny; iy++)
    for (int ix = 0; ix < L.nx; ix++)
      for (int k = 0; k < L.na; k++)
        out[w++] = response_sum(grid, g->data_size, L.base[iy * L.nx + ix], lut + (size_t)k * n, n);
  free(L.base);
  return B2S_OK;
}

/* ScanMatcher::ComputePositionalCovariance (Mapper.cpp:535-630).  probs = m_pSearchSpaceProbs (side x side,
 * width step = AlignValue(side, 8)), probs_off its converter offset. */
static int positional_covariance(const b2s_grid_info *g, double resolution_param, const double *probs,
                                 const double probs_off[2], const double best_pose[3], double best,
                                 const double center[3], const b2s_search *s, double cov[9]) {
  double scale = 1.0 / resolution_param;
  int pstep = (g->search_side + 7) & ~7;
  memset(cov, 0, 9 * sizeof(double));
  cov[0] = cov[4] = cov[8] = 1.0; /* SetToIdentity */
  if (best < KT_TOLERANCE) {
    cov[0] = MAX_VARIANCE; cov[4] = MAX_VARIANCE;
    cov[8] = 4 * (s->angle_res * s->angle_res);
    return B2S_OK;
  }
  double axx = 0, axy = 0, ayy = 0, norm = 0;
  double dx = best_pose[0] - center[0], dy = best_pose[1] - center[1];
  double off_x = s->offset_x, off_y = s->offset_y;
  int nx = orc_n_steps(off_x, s->res_x), ny = orc_n_steps(off_y, s->res_y);
  double start_x = -off_x, start_y = -off_y;
  for (int iy = 0; iy < ny; iy++) {
    double y = start_y + (uint32_t)iy * s->res_y;
    for (int ix = 0; ix < nx; ix++) {
      double x = start_x + (uint32_t)ix * s->res_x;
      int32_t px = world_to_grid_1(center[0] + x, probs_off[0], scale);
      int32_t py = world_to_grid_1(center[1] + y, probs_off[1], scale);
      if (!(px >= 0 && px < g->search_side && py >= 0 && py < g->search_side)) return B2S_ERR_OUT_OF_RANGE;
      double response = probs[px + py * pstep];
      if (response >= (best - 0.1)) {
        norm += response;
        axx += ((x - dx) * (x - dx) * response);
        axy += ((x - dx) * (y - dy) * response);
        ayy += ((y - dy) * (y - dy) * response);
      }
    }
  }
  if (norm > KT_TOLERANCE) {
    double vxx = axx / norm, vxy = axy / norm, vyy = ayy / norm;
    double vthth = 4 * (s->angle_res * s->angle_res);
    double min_xx = 0.1 * (s->res_x * s->res_x), min_yy = 0.1 * (s->res_y * s->res_y);
    vxx = dmax(vxx, min_xx);
    vyy = dmax(vyy, min_yy);
    double mult = 1.0 / best;
    cov[0] = vxx * mult; cov[1] = vxy * mult; cov[3] = vxy * mult; cov[4] = vyy * mult;
    cov[8] = vthth;
  }
  if (double_equal(cov[0], 0.0)) cov[0] = MAX_VARIANCE;
  if (double_equal(cov[4], 0.0)) cov[4] = MAX_VARIANCE;
  return B2S_OK;
}

/* ScanMatcher::ComputeAngularCovariance (Mapper.cpp:641-692) */
static int angular_covariance(const b2s_grid_info *g, double resolution_param, const double grid_off[2],
                              const uint8_t *grid, const int32_t *lut, int n, const double best_pose[3], double best,
                              const double center[3], const b2s_search *s, double cov[9]) {
  double scale = 1.0 / resolution_param;
  double best_angle = normalize_angle_difference(best_pose[2], center[2]);
  int32_t gx = world_to_grid_1(best_pose[0], grid_off[0], scale) + g->roi_x;
  int32_t gy = world_to_grid_1(best_pose[1], grid_off[1], scale) + g->roi_y;
  if (!(gx >= 0 && gx < g->width && gy >= 0 && gy < g->height)) return B2S_ERR_OUT_OF_RANGE;
  int32_t base = gx + gy * g->width_step;
  int na = orc_n_steps(s->angle_offset, s->angle_res); /* "* 2" vs "* 2.0": same double arithmetic */
  double start = center[2] - s->angle_offset;
  double norm = 0.0, acc = 0.0;
  for (int k = 0; k < na; k++) {
    double angle = start + (uint32_t)k * s->angle_res;
    double response = (double)response_sum(grid, g->data_size, base, lut + (size_t)k * n, n);
    response /= ((uint32_t)n * GRID_OCCUPIED);
    if (response >= (best - 0.1)) {
      norm += response;
      acc += ((angle - best_angle) * (angle - best_angle) * response);
    }
  }
  if (norm > KT_TOLERANCE) {
    if (acc < KT_TOLERANCE) acc = s->angle_res * s->angle_res;
    acc /= norm;
  } else {
    acc = 1000 * (s->angle_res * s->angle_res);
  }
  cov[8] = acc;
  return B2S_OK;
}

/* ScanMatcher::CorrelateScan (Mapper.cpp:309-523).
 * ranges/pts_xy/sensor_pose describe the scan being matched; result->cov is IN/OUT when s->fine.
 * sums_out (optional, [ny][nx][na]) receives the integer response numerators. */
int orc_correlate_scan(const b2s_matcher_params *p, const b2s_grid_info *g, const double grid_off[2],
                       const uint8_t *grid, const double *ranges, const double *pts_xy, int n,
                       const double sensor_pose[3], const double center[3], const b2s_search *s,
                       b2s_match_result *result, int32_t *sums_out) {
  int na = orc_n_steps(s->angle_offset, s->angle_res);
  int32_t *lut = (int32_t *)malloc(sizeof(int32_t) * (size_t)na * n);
  orc_compute_offsets(g, p->resolution, grid_off, ranges, pts_xy, n, sensor_pose, center[2], s->angle_offset,
                      s->angle_res, lut);
  sweep_layout L;
  int rc = sweep_bases(g, p->resolution, grid_off, center, s, &L);
  if (rc) {
    free(lut);
    result->status = rc;
    return rc;
  }
  double scale = 1.0 / p->resolution;
  int pstep = (g->search_side + 7) & ~7;
  double *probs = NULL;
  double probs_off[2] = {0, 0};
  if (!s->fine) {
    probs = (double *)calloc((size_t)pstep * g->search_side, sizeof(double)); /* Clear (Mapper.cpp:329) */
    probs_off[0] = center[0] - s->offset_x;                                   /* Mapper.cpp:332-333 */
    probs_off[1] = center[1] - s->offset_y;
  }
  size_t total = (size_t)L.nx * L.ny * L.na;
  double *resp = (double *)malloc(sizeof(double) * total);
  double *pose = (double *)malloc(sizeof(double) * 3 * total);
  double start_x = -s->offset_x, start_y = -s->offset_y;
  size_t w = 0;
  for (int iy = 0; iy < L.ny; iy++) {
    double y = start_y + (uint32_t)iy * s->res_y;
    double new_y = center[1] + y;
    double sq_y = y * y;
    for (int ix = 0; ix < L.nx; ix++) {
      double x = start_x + (uint32_t)ix * s->res_x;
      double new_x = center[0] + x;
      double sq_x = x * x;
      int32_t base = L.base[iy * L.nx + ix];
      double start_angle = center[2] - s->angle_offset;
      for (int k = 0; k < L.na; k++, w++) {
        double angle = start_angle + (uint32_t)k * s->angle_res;
        int32_t isum = response_sum(grid, g->data_size, base, lut + (size_t)k * n, n);
        if (sums_out) sums_out[w] = isum;
        double response = (double)isum;
        response /= ((uint32_t)n * GRID_OCCUPIED); /* Mapper.cpp:852 */
        if (s->do_penalize && !double_equal(response, 0.0)) {
          double sq_d = sq_x + sq_y;
          double dpen = 1.0 - (DISTANCE_PENALTY_GAIN * sq_d / p->distance_variance_penalty);
          dpen = dmax(dpen, p->minimum_distance_penalty);
          double sq_a = (angle - center[2]) * (angle - center[2]);
          double apen = 1.0 - (ANGLE_PENALTY_GAIN * sq_a / p->angle_variance_penalty);
          apen = dmax(apen, p->minimum_angle_penalty);
          response *= (dpen * apen);
        }
        resp[w] = response;
        pose[3 * w] = new_x; pose[3 * w + 1] = new_y; pose[3 * w + 2] = orc_normalize_angle(angle);
      }
    }
  }
  /* best response + per-cell maxima (Mapper.cpp:430-451) */
  double best = -1;
  rc = B2S_OK;
  for (size_t i = 0; i < total && rc == B2S_OK; i++) {
    best = dmax(best, resp[i]);
    if (!s->fine) {
      int32_t px = world_to_grid_1(pose[3 * i], probs_off[0], scale);
      int32_t py = world_to_grid_1(pose[3 * i + 1], probs_off[1], scale);
      if (!(px >= 0 && px < g->search_side && py >= 0 && py < g->search_side)) {
        rc = B2S_ERR_OUT_OF_RANGE; /* GetDataPointer -> GridIndex throws (Karto.h:4553-4557) */
        break;
      }
      double *ptr = probs + px + (size_t)py * pstep;
      *ptr = dmax(resp[i], *ptr);
    }
  }
  /* average of all poses tied with the best (Mapper.cpp:455-487) */
  double ax = 0, ay = 0, thx = 0, thy = 0;
  int32_t count = 0;
  if (rc == B2S_OK) {
    for (size_t i = 0; i < total; i++) {
      if (double_equal(resp[i], best)) {
        ax += pose[3 * i];
        ay += pose[3 * i + 1];
        thx += cos(pose[3 * i + 2]);
        thy += sin(pose[3 * i + 2]);
        count++;
      }
    }
    if (count > 0) {
      ax /= count; ay /= count; thx /= count; thy /= count;
    } else {
      rc = B2S_ERR_NO_BEST_POSE;
    }
  }
  if (rc == B2S_OK) {
    double avg[3] = {ax, ay, atan2(thy, thx)};
    if (!s->fine)
      rc = positional_covariance(g, p->resolution, probs, probs_off, avg, best, center, s, result->cov);
    else
      rc = angular_covariance(g, p->resolution, grid_off, grid, lut, n, avg, best, center, s, result->cov);
    if (rc == B2S_OK) {
      result->pose[0] = avg[0]; result->pose[1] = avg[1]; result->pose[2] = avg[2];
      if (best > 1.0) best = 1.0;
      result->response = best;
      result->tie_count = count;
    }
  }
  result->status = rc;
  free(lut); free(L.base); free(resp); free(pose); free(probs);
  return rc;
}

/* ScanMatcher::MatchScan (Mapper.cpp:184-291) for one scan + n_base base scans given as ranges/poses.
 * grid_out (optional, data_size bytes) / grid_off_out (optional) return the correlation grid it built. */
int orc_match_scan(const b2s_matcher_params *p, const b2s_laser *l, const double *ranges, const double robot_pose[3],
                   int n_base, const double *base_ranges, const double *base_poses, int do_penalize, int do_refine,
                   b2s_match_result *result, uint8_t *grid_out, double *grid_off_out) {
  b2s_grid_info g;
  int rc = orc_matcher_layout(p, &g);
  if (rc) {
    result->status = rc;
    return rc;
  }
  int n = l->n_readings;
  double sp[3];
  orc_sensor_pose(robot_pose, l->offset_pose, sp);
  memset(result, 0, sizeof(*result));
  if (n == 0) { /* Mapper.cpp:199-209 */
    result->pose[0] = sp[0]; result->pose[1] = sp[1]; result->pose[2] = sp[2];
    result->cov[0] = MAX_VARIANCE; result->cov[4] = MAX_VARIANCE;
    result->cov[8] = 4 * (p->coarse_angle_resolution * p->coarse_angle_resolution);
    result->response = 0.0;
    return B2S_OK;
  }
  double off[2];
  orc_grid_offset(&g, p->resolution, sp, off);
  uint8_t *grid = (uint8_t *)malloc((size_t)g.data_size);
  double *pts = (double *)malloc(sizeof(double) * 2 * (size_t)n);
  orc_add_scans(p, l, &g, off, grid, n_base, base_ranges, base_poses, sp);
  orc_point_readings(l, ranges, robot_pose, pts);

  double resolution = 1.0 / (1.0 / p->resolution);
  b2s_search coarse;
  coarse.offset_x = 0.5 * ((double)g.search_side - 1) * resolution; /* Mapper.cpp:228-230 */
  coarse.offset_y = coarse.offset_x;
  coarse.res_x = 2 * resolution; /* Mapper.cpp:233-234 */
  coarse.res_y = 2 * resolution;
  coarse.angle_offset = p->coarse_search_angle_offset;
  coarse.angle_res = p->coarse_angle_resolution;
  coarse.do_penalize = do_penalize;
  coarse.fine = 0;
  rc = orc_correlate_scan(p, &g, off, grid, ranges, pts, n, sp, sp, &coarse, result, NULL);
  if (rc == B2S_OK && p->use_response_expansion) { /* Mapper.cpp:242-272 */
    if (double_equal(result->response, 0.0)) {
      double new_off = p->coarse_search_angle_offset;
      for (uint32_t i = 0; i < 3 && rc == B2S_OK; i++) {
        new_off += 20 * 0.01745329251994329577; /* math::DegreesToRadians(20) */
        coarse.angle_offset = new_off;
        rc = orc_correlate_scan(p, &g, off, grid, ranges, pts, n, sp, sp, &coarse, result, NULL);
        if (rc == B2S_OK && double_equal(result->response, 0.0) == 0) break;
      }
    }
  }
  if (rc == B2S_OK && do_refine) { /* Mapper.cpp:274-282 */
    b2s_search fine;
    fine.offset_x = coarse.res_x * 0.5;
    fine.offset_y = coarse.res_y * 0.5;
    fine.res_x = resolution;
    fine.res_y = resolution;
    fine.angle_offset = 0.5 * p->coarse_angle_resolution;
    fine.angle_res = p->fine_search_angle_offset;
    fine.do_penalize = do_penalize;
    fine.fine = 1;
    double center[3] = {result->pose[0], result->pose[1], result->pose[2]};
    rc = orc_correlate_scan(p, &g, off, grid, ranges, pts, n, sp, center, &fine, result, NULL);
  }
  if (grid_out) memcpy(grid_out, grid, (size_t)g.data_size);
  if (grid_off_out) { grid_off_out[0] = off[0]; grid_off_out[1] = off[1]; }
  free(grid); free(pts);
  result->status = rc;
  return rc;
}

/* ------------------------------------------------------------------ K2c: karto::OccupancyGrid */

/* OccupancyGrid::ComputeDimensions (Karto.h:5804-5822) */
void orc_occ_dimensions(const b2s_laser *l, int n_scans, const double *ranges, const double *poses,
                        double resolution, b2s_occ_grid_info *info) {
  double mnx = 999999999999999999.99999, mny = mnx, mxx = -mnx, mxy = -mnx;
  for (int s = 0; s < n_scans; s++) {
    double bb[4];
    orc_scan_bbox(l, ranges + (size_t)s * l->n_readings, poses + 3 * (size_t)s, bb);
    /* BoundingBox2::Add(box) = Add(min); Add(max) (Karto.h:2824-2828) */
    if (bb[0] < mnx) mnx = bb[0];
    if (bb[1] < mny) mny = bb[1];
    if (bb[0] > mxx) mxx = bb[0];
    if (bb[1] > mxy) mxy = bb[1];
    if (bb[2] < mnx) mnx = bb[2];
    if (bb[3] < mny) mny = bb[3];
    if (bb[2] > mxx) mxx = bb[2];
    if (bb[3] > mxy) mxy = bb[3];
  }
  double scale = 1.0 / resolution;
  info->width = (int32_t)orc_round((mxx - mnx) * scale);
  info->height = (int32_t)orc_round((mxy - mny) * scale);
  info->width_step = (info->width + 7) & ~7;
  info->data_size = info->width_step * info->height;
  info->offset[0] = mnx;
  info->offset[1] = mny;
  info->resolution = resolution;
  info->cell_visits = 0;
}

/* Grid<T>::TraceLine (Karto.h:4680-4745) incrementing pass[]; returns the number of in-grid cells touched */
static uint64_t trace_line(int w, int h, int step, uint32_t *pass, int x0, int y0, int x1, int y1) {
  uint64_t touched = 0;
  int steep = abs(y1 - y0) > abs(x1 - x0);
  int t;
  if (steep) {
    t = x0; x0 = y0; y0 = t;
    t = x1; x1 = y1; y1 = t;
  }
  if (x0 > x1) {
    t = x0; x0 = x1; x1 = t;
    t = y0; y0 = y1; y1 = t;
  }
  int dx = x1 - x0, dy = abs(y1 - y0), error = 0, ystep, y = y0;
  ystep = (y0 < y1) ? 1 : -1;
  for (int x = x0; x <= x1; x++) {
    int px = steep ? y : x, py = steep ? x : y;
    error += dy;
    if (2 * error >= dx) {
      y += ystep;
      error -= dx;
    }
    if (px >= 0 && px < w && py >= 0 && py < h) {
      pass[px + py * step]++;
      touched++;
    }
  }
  return touched;
}

int orc_trace_line_cells(int w, int h, int x0, int y0, int x1, int y1, int32_t *out_xy, int cap) {
  int n = 0;
  int steep = abs(y1 - y0) > abs(x1 - x0);
  int t;
  if (steep) {
    t = x0; x0 = y0; y0 = t;
    t = x1; x1 = y1; y1 = t;
  }
  if (x0 > x1) {
    t = x0; x0 = x1; x1 = t;
    t = y0; y0 = y1; y1 = t;
  }
  int dx = x1 - x0, dy = abs(y1 - y0), error = 0, ystep, y = y0;
  ystep = (y0 < y1) ? 1 : -1;
  for (int x = x0; x <= x1; x++) {
    int px = steep ? y : x, py = steep ? x : y;
    error += dy;
    if (2 * error >= dx) {
      y += ystep;
      error -= dx;
    }
    if (px >= 0 && px < w && py >= 0 && py < h) {
      if (n < cap) { out_xy[2 * n] = px; out_xy[2 * n + 1] = py; }
      n++;
    }
  }
  return n;
}

/* OccupancyGrid::CreateFromScans -> AddScan -> RayTrace -> Update (Karto.h:5828-5990).
 * pass/hit/cells are info->data_size long. */
void orc_occ_create_from_scans(const b2s_laser *l, int n_scans, const double *ranges, const double *poses,
                               b2s_occ_grid_info *info, uint32_t *pass, uint32_t *hit, uint8_t *cells) {
  int n = l->n_readings;
  int w = info->width, h = info->height, step = info->width_step;
  double scale = 1.0 / info->resolution;
  memset(pass, 0, sizeof(uint32_t) * (size_t)info->data_size);
  memset(hit, 0, sizeof(uint32_t) * (size_t)info->data_size);
  double *pts = (double *)malloc(sizeof(double) * 2 * (size_t)n);
  uint64_t visits = 0;
  for (int s = 0; s < n_scans; s++) {
    const double *r = ranges + (size_t)s * n;
    double sp[3];
    orc_sensor_pose(poses + 3 * (size_t)s, l->offset_pose, sp);
    orc_point_readings(l, r, poses + 3 * (size_t)s, pts);
    for (int i = 0; i < n; i++) {
      double px = pts[2 * i], py = pts[2 * i + 1];
      double rr = r[i];
      int end_valid = rr < (l->range_threshold - KT_TOLERANCE);
      if (rr <= l->min_range || rr >= l->max_range || isnan(rr)) continue;
      if (rr >= l->range_threshold) {
        double ratio = l->range_threshold / rr;
        double dx = px - sp[0], dy = py - sp[1];
        px = sp[0] + ratio * dx;
        py = sp[1] + ratio * dy;
      }
      int32_t fx = world_to_grid_1(sp[0], info->offset[0], scale), fy = world_to_grid_1(sp[1], info->offset[1], scale);
      int32_t tx = world_to_grid_1(px, info->offset[0], scale), ty = world_to_grid_1(py, info->offset[1], scale);
      visits += trace_line(w, h, step, pass, fx, fy, tx, ty);
      if (end_valid && tx >= 0 && tx < w && ty >= 0 && ty < h) {
        pass[tx + ty * step]++;
        hit[tx + ty * step]++;
        visits += 2;
      }
    }
  }
  info->cell_visits = visits;
  /* Update / UpdateCell (Karto.h:5953-5990): MinPassThrough = 2, OccupancyThreshold = 0.1 (Karto.h:5632-5633) */
  memset(cells, 0, (size_t)info->data_size);
  for (int32_t i = 0; i < info->data_size; i++) {
    if (pass[i] > 2u) {
      double ratio = (double)hit[i] / (double)pass[i];
      cells[i] = ratio > 0.1 ? GRID_OCCUPIED : GRID_FREE;
    }
  }
  free(pts);
}
