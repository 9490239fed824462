// lesson4 Hector grid arithmetic shared by the single-map handle (hector_map.cu) and the processor (hector_slam.cu).
// Each function below is the one restatement of the reference function it cites, in the reference's float32
// operation order (the library is built with -fmad=false): both handles reproduce the reference bit for bit through it.
//
// Reference paths are relative to reference/lesson4/include/lesson4/hector_mapping.
#pragma once
#include <cmath>

#include "common.cuh"

namespace b2s {

// ---- map <-> world transform ----

// GridMapBase::setMapTransformation (map/GridMapBase.h:270-286): worldTmap = AlignedScaling2f(s, s) * Translation2f(off)
// with s = 1 / cellLength, i.e. linear diag(s, s) and translation s * off; mapTworld is its Affine inverse in Eigen's
// cofactor form.
struct MapTransform {
  float tw_lin, tw_tx, tw_ty;  // world -> map
  float wt_lin, wt_tx, wt_ty;  // map -> world
};
inline MapTransform map_transform(float cell_length, float off_x, float off_y) {
  MapTransform t;
  const float scale_to_map = 1.0f / cell_length;
  t.tw_lin = scale_to_map;
  t.tw_tx = scale_to_map * off_x;
  t.tw_ty = scale_to_map * off_y;
  const float det = t.tw_lin * t.tw_lin - 0.0f * 0.0f, invdet = 1.0f / det, i01 = -0.0f * invdet;
  t.wt_lin = t.tw_lin * invdet;
  t.wt_tx = -(t.wt_lin * t.tw_tx + i01 * t.tw_ty);
  t.wt_ty = -(i01 * t.tw_tx + t.wt_lin * t.tw_ty);
  return t;
}

// getMapCoordsPose (map/GridMapBase.h:238-242), position part: the heading passes through unchanged
__host__ __device__ __forceinline__ void get_map_coords(const MapTransform &t, float wx, float wy, float &mx, float &my) {
  mx = (t.tw_lin * wx + 0.0f * wy) + t.tw_tx;
  my = (0.0f * wx + t.tw_lin * wy) + t.tw_ty;
}

// getWorldCoordsPose (map/GridMapBase.h:229-233), position part
__host__ __device__ __forceinline__ void get_world_coords(const MapTransform &t, float mx, float my, float &wx, float &wy) {
  wx = (t.wt_lin * mx + (-0.0f) * my) + t.wt_tx;
  wy = ((-0.0f) * mx + t.wt_lin * my) + t.wt_ty;
}

// ---- OccGridMapBase::updateByScan (map/OccGridMapBase.h:118-168) ----
// poseTransform = Translation2f(mx, my) * Rotation2Df(theta) with c, s = cos / sin of theta.

// begin cell: Vector2i(poseTransform * origo + 0.5f), the int constructor truncates (:130-135)
__host__ __device__ __forceinline__ int2 begin_cell(float c, float s, float mx, float my, float ox, float oy) {
  const float bx = (c * ox + (-s) * oy) + mx, by = (s * ox + c * oy) + my;
  return make_int2((int)(bx + 0.5f), (int)(by + 0.5f));
}

// end cell of one beam: (poseTransform * p + 0.5f).cast<int>(), truncation (:147-154)
__device__ __forceinline__ int2 end_cell(float c, float s, float mx, float my, float px, float py) {
  const float ex = __fadd_rn(__fadd_rn(__fmul_rn(c, px), __fmul_rn(-s, py)), mx);
  const float ey = __fadd_rn(__fadd_rn(__fmul_rn(s, px), __fmul_rn(c, py)), my);
  return make_int2((int)__fadd_rn(ex, 0.5f), (int)__fadd_rn(ey, 0.5f));
}

// end cell of one beam in updateByScanJustOnce (:175-217), the lesson4 make-map variant: begin + (int)round(p / 0.05)
// on the raw point in metres (float / double literal -> double, ::round, (int)), whatever the map's cell size
__device__ __forceinline__ int2 just_once_end_cell(int bx, int by, float px, float py) {
  return make_int2(bx + cast_i32(round((double)px / 0.05)), by + cast_i32(round((double)py / 0.05)));
}

// updateLineBresenhami's set-up (:220-258): the line is drawn iff begin != end and both cells are inside the map.
// bresenham2D then visits da cells from the start (the end cell excluded), see bresenham_offset.
struct BresenhamLine {
  bool ok;
  int x0, y0, x1, y1;
  unsigned int da, db;  // major / minor axis lengths
  int err0, off_a, off_b;  // initial error, flat offsets of a major / minor step
};
__device__ __forceinline__ BresenhamLine bresenham_line(int x0, int y0, int2 end, int sx, int sy) {
  BresenhamLine L;
  L.x0 = x0; L.y0 = y0;
  L.x1 = end.x; L.y1 = end.y;
  L.ok = !(L.x0 == L.x1 && L.y0 == L.y1);
  if ((L.x0 < 0) || (L.x0 >= sx) || (L.y0 < 0) || (L.y0 >= sy)) L.ok = false;
  if ((L.x1 < 0) || (L.x1 >= sx) || (L.y1 < 0) || (L.y1 >= sy)) L.ok = false;
  const int dx = L.x1 - L.x0, dy = L.y1 - L.y0;
  const unsigned int adx = (unsigned int)abs(dx), ady = (unsigned int)abs(dy);
  const int odx = dx > 0 ? 1 : -1, ody = (dy > 0 ? 1 : -1) * sx;  // util::sign: sign(0) = -1
  if (adx >= ady) { L.da = adx; L.db = ady; L.err0 = (int)(adx / 2); L.off_a = odx; L.off_b = ody; }
  else { L.da = ady; L.db = adx; L.err0 = (int)(ady / 2); L.off_a = ody; L.off_b = odx; }
  return L;
}

// bresenham2D (:262-300) in closed form: the flat offset of the cell of step k < da, `start` being the begin cell's.
// After k major steps the minor axis has stepped floor((err0 + k * db) / da) times.
__device__ __forceinline__ int bresenham_offset(const BresenhamLine &L, int start, unsigned int k) {
  const unsigned int inc = (unsigned int)(((unsigned long long)L.err0 + (unsigned long long)k * L.db) / L.da);
  return start + (int)k * L.off_a + (int)inc * L.off_b;
}

// ---- scan matching ----

// interpMapValueWithDerivatives (map/OccGridMapUtil.h:139-228).  Its bounds test: setMapCellDims keeps dims - 2.
__device__ __forceinline__ bool interp_inside(int sx, int sy, float x, float y) {
  const float lim_x = (float)sx - 2.0f, lim_y = (float)sy - 2.0f;
  return !(x < 0.0f || x > lim_x || y < 0.0f || y > lim_y);
}
// Its bilinear value and gradient from the probabilities of cells (x, y), (x+1, y), (x, y+1), (x+1, y+1) and the
// fractional position (fx, fy) inside cell (x, y): out = {value, d/dx, d/dy}.
__device__ __forceinline__ void interp_finish(float i0, float i1, float i2, float i3, float fx, float fy, float out[3]) {
  const float dx1 = i0 - i1, dx2 = i2 - i3, dy1 = i0 - i2, dy2 = i1 - i3;
  const float xfi = 1.0f - fx, yfi = 1.0f - fy;
  out[0] = ((i0 * xfi + i1 * fx) * yfi) + ((i2 * xfi + i3 * fx) * fy);
  out[1] = -((dx1 * yfi) + (dx2 * fy));
  out[2] = -((dy1 * xfi) + (dy2 * fx));
}

// Matrix3f::inverse() * v (estimateTransformationLogLh, matcher/ScanMatcher.h:107-141)
__device__ __forceinline__ void inv3_mul(const float m[9], const float v[3], float out[3]) {
  const float c00 = m[4] * m[8] - m[5] * m[7], c10 = m[5] * m[6] - m[3] * m[8], c20 = m[3] * m[7] - m[4] * m[6];
  const float det = c00 * m[0] + (c10 * m[1] + c20 * m[2]);  /* Eigen's unrolled 3-term redux: a0 + (a1 + a2) */
  const float invdet = 1.0f / det;
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

// util::normalize_angle (util/UtilFunctions.h:36-48): fmod(fmod(a, 2pi) + 2pi, 2pi) in double, float result, then
// `a -= 2.0f*M_PI` (promoted to double) above pi.  Out of line: the double fmod expansion is large, and the Gauss-Newton
// loops that call it must stay inside the instruction cache.
inline __device__ __noinline__ float util_normalize_angle(float e2) {
  const double two_pi = 2.0f * 3.14159265358979323846;
  const double d = (double)e2;
  double r;
  if (fabs(d) < two_pi) {
    // fmod(d, 2pi) = d here, and for x = d + 2pi in (0, 4pi): fmod(x, 2pi) = x - 2pi when x >= 2pi (exact: Sterbenz), else x.
    // Bit for bit the reference's two fmod calls, without the two software remainder loops (tests/normalize_angle_check.c).
    const double x = d + two_pi;
    r = x >= two_pi ? x - two_pi : x;
  } else {
    r = fmod(fmod(d, two_pi) + two_pi, two_pi);
  }
  float a = (float)r;
  if ((double)a > 3.14159265358979323846) a = (float)((double)a - two_pi);
  return a;
}

// ---- log-odds cells (map/GridMapLogOdds.h) ----

// GridMapLogOddsFunctions::probToLogOdds (:153-157), as setUpdateFreeFactor / setUpdateOccupiedFactor use it (:98-102).
// The reference's unqualified log(odds) is the C library's double log, rounded to float: prob_to_log_odds.  The
// single-map handle takes logf instead: prob_to_log_odds_logf.  The two agree on the factors the tests use (0.4, 0.6,
// 0.9), but a factor whose double logarithm rounds differently from logf gives that handle a different log-odds step.
inline float prob_to_log_odds(float prob) {
  const float odds = prob / (1.0f - prob);
  return (float)log((double)odds);
}
inline float prob_to_log_odds_logf(float prob) {
  const float odds = prob / (1.0f - prob);
  return logf(odds);
}

// GridMapLogOddsFunctions::getGridProbability (:136-140) as the processor computes it: the unqualified exp() is the C
// library's double exp, rounded to float (the device's double exp; tests/device_math_check.cu compares every float in
// [-128, 64] against the C library).
__host__ __device__ __forceinline__ float log_odds_prob(float lo) {
  const float odds = (float)exp((double)lo);
  return odds / (odds + 1.0f);
}

// HectorMappingRos::publishMap (lesson4/src/hector_mapping/hector_slam.cc:254-317): free -> 0, occupied -> 100, else -1.
__device__ __forceinline__ int8_t hector_ros_cell(float v) { return v < 0.0f ? 0 : (v > 0.0f ? 100 : -1); }

// `static`: each translation unit gets its own copy, the library exports nothing from here.
static __global__ void k_hector_ros(const float *__restrict__ lo, int n, int8_t *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = hector_ros_cell(lo[i]);
}

}  // namespace b2s
