// lesson4 GMapping grid arithmetic shared by the map handle (gmapping_map.cu) and the make-map node call
// (lesson4_node_maps.cu).  Each function below is the one restatement of the reference code it cites, in the
// reference's double operation order (the library is built with -fmad=false).
//
// Reference paths are relative to reference/lesson4.
#pragma once
#include <cmath>

#include "common.cuh"

namespace b2s {

// Map::world2map, one axis (include/lesson4/gmapping/grid/map.h:171-174)
__device__ __forceinline__ int gm_world2map(double w, double c, double delta, int half) {
  return cast_i32(round((w - c) / delta)) + half;
}

struct GmRay {
  bool valid, hit;
  int p1x, p1y;
  double hx, hy;
};

// One beam of GMapping::ComputeMap (src/gmapping/gmapping.cc:186-219) from the laser at (lx, ly) with heading 0: the
// range filter, the clip to max_use, the hit point and its cell.  unit() gives the beam's (cos, sin); it is called
// only for a kept beam.
template <class Unit>
__device__ __forceinline__ GmRay gm_ray(double d, Unit unit, double lx, double ly, double cx, double cy, double delta,
                                        int sx2, int sy2, double max_range, double max_use) {
  GmRay r;
  r.valid = !(d > max_range || d == 0.0 || !isfinite(d));  // gmapping.cc:190-191
  r.hit = false; r.p1x = r.p1y = 0; r.hx = r.hy = 0;
  if (!r.valid) return r;
  if (d > max_use) d = max_use;
  const double2 u = unit();
  r.hx = __dadd_rn(lx, __dmul_rn(d, u.x));
  r.hy = __dadd_rn(ly, __dmul_rn(d, u.y));
  r.p1x = gm_world2map(r.hx, cx, delta, sx2);
  r.p1y = gm_world2map(r.hy, cy, delta, sy2);
  r.hit = d < max_use;  // gmapping.cc:214
  return r;
}

// GridLineTraversal::gridLine (include/lesson4/gmapping/grid/gridlinetraversal.h:27-207) from p0 to p1 in closed form.
// The canonical traversal starts at the endpoint with the smaller dominant coordinate (the start wins ties); its step k
// (0 <= k <= dmaj) is on the minor axis j(k) = floor((2*k*dmin + dmaj) / (2*dmaj)) cells away from its first cell.
struct GmLine {
  bool xmajor;
  int b_maj, b_min, step_min;
  long long dmaj, dmin, k_end;  // k_end: the step at which the traversal sits on p1
};
__device__ __forceinline__ GmLine gm_line(int p0x, int p0y, int p1x, int p1y) {
  GmLine L;
  const int dx = abs(p1x - p0x), dy = abs(p1y - p0y);
  L.xmajor = dy <= dx;  // gridlinetraversal.h:44
  const int s_maj = L.xmajor ? p0x : p0y, e_maj = L.xmajor ? p1x : p1y;
  const int s_min = L.xmajor ? p0y : p0x, e_min = L.xmajor ? p1y : p1x;
  const bool from_end = s_maj > e_maj;
  L.b_maj = from_end ? e_maj : s_maj;
  L.b_min = from_end ? e_min : s_min;
  const int o_min = from_end ? s_min : e_min;
  L.step_min = (o_min > L.b_min) ? 1 : -1;
  L.dmaj = L.xmajor ? dx : dy;
  L.dmin = L.xmajor ? dy : dx;
  L.k_end = from_end ? 0 : L.dmaj;
  return L;
}
// the cell of step k
__device__ __forceinline__ int2 gm_line_cell(const GmLine &L, long long k) {
  const long long j = L.dmaj > 0 ? (2 * k * L.dmin + L.dmaj) / (2 * L.dmaj) : 0;
  const int maj = L.b_maj + (int)k, mn = L.b_min + L.step_min * (int)j;
  return L.xmajor ? make_int2(maj, mn) : make_int2(mn, maj);
}

// PointAccumulator::operator double (include/lesson4/gmapping/grid/map.h:27) against occ_thresh, as PublishMap
// classifies a cell (gmapping.cc:147-157): -1 unknown, 100 occupied, 0 free
__device__ __forceinline__ int8_t gm_classify(int32_t n, int32_t visits, double occ_thresh) {
  const double occ = visits ? (double)n * 1 / (double)visits : -1;
  return occ < 0 ? -1 : (occ > occ_thresh ? 100 : 0);
}

}  // namespace b2s
