// TEST INFRASTRUCTURE — not product code.
// extern "C" driver around the reference's REAL GMapping grid headers
//   reference/lesson4/include/lesson4/gmapping/grid/{map.h,gridlinetraversal.h,harray2d.h,array2d.h}, utils/point.h
// (dependency-free; gmapping.cc itself needs ROS).  GMapping::ComputeMap (src/gmapping/gmapping.cc:171-242) is
// re-assembled here around those headers with the node's ROS message replaced by plain arrays: the Bresenham lines,
// the PointAccumulator cells, the patch storage and world2map are all the reference's own code.
// Built by oracle/recipes.py into oracle/_ref/libgmapping_ref.so.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "lesson4/gmapping/grid/map.h"
#include "lesson4/gmapping/grid/gridlinetraversal.h"

using namespace gmapping;

extern "C" {

void *refg_map_create(double cx, double cy, double xmin, double ymin, double xmax, double ymax, double delta) {
  Point center(cx, cy);
  return new ScanMatcherMap(center, xmin, ymin, xmax, ymax, delta);  // gmapping.cc:135
}
void refg_map_destroy(void *h) { delete static_cast<ScanMatcherMap *>(h); }
void refg_map_size(void *h, int32_t out[2]) {
  ScanMatcherMap *m = static_cast<ScanMatcherMap *>(h);
  out[0] = m->getMapSizeX();
  out[1] = m->getMapSizeY();
}

// GMapping::ComputeMap (gmapping.cc:171-242).  lp = (laser_x, laser_y, 0) — the node uses (0,0,0).
// Returns 0, or -1 if a ray would leave the map (the reference asserts / indexes out of range there).
int refg_compute_map(void *h, const double *ranges, const double *angles, int n, double laser_x, double laser_y,
                     double max_range, double max_use_range) {
  ScanMatcherMap &map = *static_cast<ScanMatcherMap *>(h);
  std::vector<GridLineTraversalLine> line_lists;
  std::vector<Point> hit_lists;
  OrientedPoint lp(laser_x, laser_y, 0.0);
  IntPoint p0 = map.world2map(lp);
  HierarchicalArray2D<PointAccumulator>::PointSet activeArea;
  auto inside = [&](const IntPoint &p) { return p.x >= 0 && p.y >= 0 && p.x < map.getMapSizeX() && p.y < map.getMapSizeY(); };
  if (!inside(p0)) return -1;
  for (int i = 0; i < n; i++) {
    double d = ranges[i];
    if (d > max_range || d == 0.0 || !std::isfinite(d)) continue;
    if (d > max_use_range) d = max_use_range;
    Point phit = lp;
    phit.x += d * cos(angles[i]);
    phit.y += d * sin(angles[i]);
    IntPoint p1 = map.world2map(phit);
    if (!inside(p1)) return -1;
    GridLineTraversalLine line;
    GridLineTraversal::gridLine(p0, p1, &line);
    line_lists.push_back(line);
    for (int k = 0; k < line.num_points - 1; k++) activeArea.insert(map.storage().patchIndexes(line.points[k]));
    if (d < max_use_range) {
      IntPoint cp = map.storage().patchIndexes(p1);
      activeArea.insert(cp);
      hit_lists.push_back(phit);
    }
  }
  map.storage().setActiveArea(activeArea, true);
  map.storage().allocActiveArea();
  for (auto &line : line_lists)
    for (int k = 0; k < line.num_points - 1; k++) map.cell(line.points[k]).update(false, Point(0, 0));
  for (auto &hit : hit_lists) {
    IntPoint p1 = map.world2map(hit);
    map.cell(p1).update(true, hit);
  }
  return 0;
}

// per cell (index x + y*sizeX): n, visits, acc; cells in unallocated patches report the m_unknown cell (all zero)
void refg_copy(void *h, int32_t *n, int32_t *visits, float *acc_x, float *acc_y, double *occ) {
  const ScanMatcherMap &map = *static_cast<ScanMatcherMap *>(h);
  int sx = map.getMapSizeX(), sy = map.getMapSizeY();
  for (int y = 0; y < sy; y++)
    for (int x = 0; x < sx; x++) {
      const PointAccumulator &c = map.cell(IntPoint(x, y));
      size_t i = (size_t)x + (size_t)y * sx;
      if (n) n[i] = c.n;
      if (visits) visits[i] = c.visits;
      if (acc_x) acc_x[i] = c.acc.x;
      if (acc_y) acc_y[i] = c.acc.y;
      if (occ) occ[i] = (double)c;  // PointAccumulator::operator double (map.h:27)
    }
}

void refg_world2map(void *h, double x, double y, int32_t out[2]) {
  IntPoint p = static_cast<ScanMatcherMap *>(h)->world2map(Point(x, y));
  out[0] = p.x; out[1] = p.y;
}

int refg_grid_line(int x0, int y0, int x1, int y1, int32_t *out_xy, int cap) {
  GridLineTraversalLine line;
  GridLineTraversal::gridLine(IntPoint(x0, y0), IntPoint(x1, y1), &line);
  for (int i = 0; i < line.num_points && i < cap; i++) { out_xy[2 * i] = line.points[i].x; out_xy[2 * i + 1] = line.points[i].y; }
  return line.num_points;
}
}
