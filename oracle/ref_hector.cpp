/*
 * ref_hector.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * extern "C" driver around the UNMODIFIED lesson4 Hector headers, compiled where they lie under
 * reference/lesson4/include (oracle/recipes.py builds _ref/libhector_ref.so):
 *   hectorslam::GridMap  (map/GridMap.h -> OccGridMapBase.h:118-330, GridMapLogOdds.h:37-161, GridMapBase.h)
 *   HUtil (map/OccGridMapUtil.h:77-228)      ScanMatcher (matcher/ScanMatcher.h:60-141)
 *   HectorSlamProcessor  (slam_main/HectorSlamProcessor.h:81-108 -> MapRepMultiMap.h:144-191)
 * Eigen is absent from this image; the only stand-in is oracle/shim/Eigen/mini_eigen.h (fixed-size vector / 3x3 /
 * 2-D affine primitives whose semantics are listed in its header).  Every line of map-update, Bresenham, stamp,
 * log-odds, bilinear-interpolation and Gauss-Newton logic executed here is the reference's own.
 * The ref_hmap_* functions have the signatures of oracle/hector_oracle.c's orc_hmap_* so tests can swap them.
 */
#include <cmath>
#include <climits>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <sstream>
#include <vector>

#include "lesson4/hector_mapping/slam_main/HectorSlamProcessor.h"

/* the reference forward-declares ::GridMap and ::DataContainer at global scope (MapRepresentationInterface.h:32-34),
 * so the hectorslam names are spelled out rather than imported */
typedef hectorslam::GridMap HGridMap;
typedef hectorslam::DataContainer HData;
typedef hectorslam::OccGridMapUtilConfig<hectorslam::GridMap> HUtil;
typedef hectorslam::ScanMatcher<HUtil> HMatcher;
using hectorslam::HectorSlamProcessor;


namespace {
struct SilenceCout { /* the reference prints per level / per clamped step */
  std::streambuf *old;
  std::ostringstream sink;
  SilenceCout() : old(std::cout.rdbuf(sink.rdbuf())) {}
  ~SilenceCout() { std::cout.rdbuf(old); }
};

struct RefMap {
  HGridMap *map;
  HUtil *util;
  HMatcher *matcher;
};

void fill(HData &dc, const float *pts, int n, const float origo[2]) {
  dc.clear();
  dc.setOrigo(Eigen::Vector2f(origo[0], origo[1]));
  for (int i = 0; i < n; ++i) dc.add(Eigen::Vector2f(pts[2 * i], pts[2 * i + 1]));
}

void copy_map(const HGridMap &g, float *log_odds, int32_t *update_index) {
  int n = g.getSizeX() * g.getSizeY();
  for (int i = 0; i < n; ++i) {
    const LogOddsCell &c = g.getCell(i);
    if (log_odds) log_odds[i] = c.logOddsVal;
    if (update_index) update_index[i] = c.updateIndex;
  }
}
}  // namespace

extern "C" {

/* MapRepMultiMap ctor arithmetic for level 0 (MapRepMultiMap.h:58-74): offset = (res * size) * startCoords */
void *ref_hmap_create(int size_x, int size_y, float resolution, float start_x, float start_y) {
  RefMap *r = new RefMap;
  float total_x = resolution * static_cast<float>(size_x), total_y = resolution * static_cast<float>(size_y);
  r->map = new HGridMap(resolution, Eigen::Vector2i(size_x, size_y), Eigen::Vector2f(total_x * start_x, total_y * start_y));
  r->util = new HUtil(r->map);
  r->matcher = new HMatcher();
  return r;
}

void ref_hmap_destroy(void *h) {
  RefMap *r = static_cast<RefMap *>(h);
  if (!r) return;
  delete r->matcher;
  delete r->util;
  delete r->map;
  delete r;
}

void ref_hmap_set_factors(void *h, float update_free, float update_occ) {
  RefMap *r = static_cast<RefMap *>(h);
  r->map->setUpdateFreeFactor(update_free);
  r->map->setUpdateOccupiedFactor(update_occ);
}

void ref_hmap_copy(const void *h, float *log_odds, int32_t *update_index) {
  copy_map(*static_cast<const RefMap *>(h)->map, log_odds, update_index);
}

long ref_hmap_update_by_scan(void *h, const float *points, int n, const float origo[2], const float world_pose[3]) {
  RefMap *r = static_cast<RefMap *>(h);
  HData dc;
  fill(dc, points, n, origo);
  r->map->updateByScan(dc, Eigen::Vector3f(world_pose[0], world_pose[1], world_pose[2]));
  r->util->resetCachedData(); /* MapRepMultiMap::onMapUpdated (MapRepMultiMap.h:133-141) */
  return 0;
}

long ref_hmap_update_by_scan_just_once(void *h, const float *points, int n, const float origo[2]) {
  RefMap *r = static_cast<RefMap *>(h);
  HData dc;
  fill(dc, points, n, origo);
  r->map->updateByScanJustOnce(dc, Eigen::Vector3f(0.f, 0.f, 0.f));
  r->util->resetCachedData();
  return 0;
}

void ref_hmap_match_data(void *h, const float *pts, int n, const float begin_world[3], int max_iterations,
                         float out_world[3], float out_cov[9]) {
  RefMap *r = static_cast<RefMap *>(h);
  SilenceCout quiet;
  HData dc;
  const float o[2] = {0.f, 0.f};
  fill(dc, pts, n, o);
  Eigen::Matrix3f cov = Eigen::Matrix3f::Zero();
  Eigen::Vector3f res = r->matcher->matchData(Eigen::Vector3f(begin_world[0], begin_world[1], begin_world[2]), *r->util,
                                              dc, cov, max_iterations);
  for (int i = 0; i < 3; ++i) out_world[i] = res[i];
  if (n != 0)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) out_cov[3 * i + j] = cov(i, j);
}

/* GridMapLogOddsFunctions::getGridProbability (GridMapLogOdds.h:136-140) of the reference, for arbitrary log-odds values:
 * the values are planted into a scratch map's cells and read back through OccGridMapBase::getGridProbabilityMap. */
void ref_hector_grid_probabilities(const float *log_odds, int n, float *out) {
  HGridMap g(1.0f, Eigen::Vector2i(64, 64), Eigen::Vector2f(0.f, 0.f));
  for (int i = 0; i < n; i += 64 * 64) {
    const int cnt = n - i < 64 * 64 ? n - i : 64 * 64;
    for (int j = 0; j < cnt; ++j) g.getCell(j).logOddsVal = log_odds[i + j];
    for (int j = 0; j < cnt; ++j) out[i + j] = g.getGridProbabilityMap(j);
  }
}

/* Bresenham cell list of OccGridMapBase::updateLineBresenhami as the map sees it: run one line on a scratch map and
 * report which cells were freed / occupied (update index stamps), for the per-segment cell-set tests. */
int ref_hector_line_cells(int size, int x0, int y0, int x1, int y1, int32_t *free_cells, int32_t *n_free, int32_t *occ_cell) {
  HGridMap g(1.0f, Eigen::Vector2i(size, size), Eigen::Vector2f(0.f, 0.f));
  HData dc;
  dc.setOrigo(Eigen::Vector2f((float)x0, (float)y0));
  dc.add(Eigen::Vector2f((float)x1, (float)y1));
  /* world == map for resolution 1 and zero offset; pose 0 */
  g.updateByScan(dc, Eigen::Vector3f(0.f, 0.f, 0.f));
  int nf = 0;
  *occ_cell = -1;
  for (int i = 0; i < size * size; ++i) {
    const LogOddsCell &c = g.getCell(i);
    if (c.updateIndex < 0) continue;
    if (c.logOddsVal > 0.f) *occ_cell = i;
    else if (c.logOddsVal < 0.f) free_cells[nf++] = i;
  }
  *n_free = nf;
  return 0;
}

/* ---- the whole lesson4 front end: HectorSlamProcessor::update = multi-level matchData + updateByScan ---- */
void *ref_hproc_create(float resolution, int size_x, int size_y, float start_x, float start_y, int levels,
                       float update_free, float update_occ, float min_dist, float min_angle) {
  SilenceCout quiet;
  HectorSlamProcessor *p = new HectorSlamProcessor(resolution, size_x, size_y, Eigen::Vector2f(start_x, start_y), levels);
  p->setUpdateFactorFree(update_free);
  p->setUpdateFactorOccupied(update_occ);
  p->setMapUpdateMinDistDiff(min_dist);
  p->setMapUpdateMinAngleDiff(min_angle);
  return p;
}

void ref_hproc_destroy(void *h) { delete static_cast<HectorSlamProcessor *>(h); }

/* points are in level-0 map-cell units (hector_slam.cc scales by getScaleToMap()), pose hint in world metres */
void ref_hproc_update(void *h, const float *pts, int n, const float origo[2], const float pose_hint[3],
                      int map_without_matching, float out_pose[3], float out_cov[9]) {
  HectorSlamProcessor *p = static_cast<HectorSlamProcessor *>(h);
  SilenceCout quiet;
  HData dc;
  fill(dc, pts, n, origo);
  p->update(dc, Eigen::Vector3f(pose_hint[0], pose_hint[1], pose_hint[2]), map_without_matching != 0);
  const Eigen::Vector3f &r = p->getLastScanMatchPose();
  for (int i = 0; i < 3; ++i) out_pose[i] = r[i];
  if (!map_without_matching && out_cov) {
    const Eigen::Matrix3f &c = p->getLastScanMatchCovariance();
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) out_cov[3 * i + j] = c(i, j);
  }
}

int ref_hproc_level_dims(void *h, int level, int dims[2]) {
  HectorSlamProcessor *p = static_cast<HectorSlamProcessor *>(h);
  if (level < 0 || level >= p->getMapLevels()) return -1;
  dims[0] = p->getGridMap(level).getSizeX();
  dims[1] = p->getGridMap(level).getSizeY();
  return 0;
}

void ref_hproc_copy_level(void *h, int level, float *log_odds, int32_t *update_index) {
  copy_map(static_cast<HectorSlamProcessor *>(h)->getGridMap(level), log_odds, update_index);
}

} /* extern "C" */
