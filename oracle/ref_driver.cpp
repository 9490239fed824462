// TEST INFRASTRUCTURE — not product code.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load the library built
// from this file.
//
// A thin extern "C" driver around the UNMODIFIED reference sources
//   reference/lesson6/lib/open_karto/src/{Karto,Mapper}.cpp
// so that Python (ctypes) can run the reference's own ScanMatcher / OccupancyGrid
// on synthetic inputs, dump its internal state (correlation grid bytes, lookup
// tables, integer response sums, pass/hit counters) and time it.  Nothing here
// restates the algorithm: every number comes out of the reference's own code.
// Built by oracle/recipes.py into oracle/_ref/libkarto_ref.so (git-ignored).
//
// Private members (ScanMatcher::AddScans / GetResponse / m_pGridLookup,
// OccupancyGrid::m_pCellPassCnt ...) are reached with the usual
// "#define private public" test trick; class layout is unaffected.

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <list>
#include <map>
#include <mutex>
#include <queue>
#include <set>
#include <shared_mutex>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#define private public
#define protected public
#include <open_karto/Mapper.h>
#undef private
#undef protected

using namespace karto;

extern "C" {

struct ref_matcher_params {
  double search_size;       // ScanMatcher::Create searchSize   (Mapper.cpp:126)
  double resolution;        //                     resolution
  double smear_deviation;   //                     smearDeviation
  double range_threshold;   //                     rangeThreshold
  // values as STORED in the Mapper (the setParam* squaring, Mapper.cpp:1919-1927,
  // is the caller's business)
  double distance_variance_penalty;
  double angle_variance_penalty;
  double fine_search_angle_offset;
  double coarse_search_angle_offset;
  double coarse_angle_resolution;
  double minimum_angle_penalty;
  double minimum_distance_penalty;
  int32_t use_response_expansion;
  int32_t _pad;
};

struct ref_laser_params {
  int32_t type;  // LaserRangeFinderType (0 = Custom, 4 = Hokuyo_UTM_30LX ...)
  int32_t _pad;
  double min_angle, max_angle, angular_resolution;
  double min_range, max_range, range_threshold;
  double offset_pose[3];
};

}  // extern "C"

namespace {

struct Session {
  Mapper* mapper = nullptr;
  LaserRangeFinder* lrf = nullptr;
  ScanMatcher* matcher = nullptr;
  std::vector<LocalizedRangeScan*> scans;
  Name name;
};

int g_session_counter = 0;

struct NullBuf : std::streambuf {
  int overflow(int c) override { return c; }
};

// the reference prints "Registering sensor" etc. on std::cout; keep test logs clean
struct CoutSilencer {
  NullBuf nb;
  std::streambuf* old;
  CoutSilencer() : old(std::cout.rdbuf(&nb)) {}
  ~CoutSilencer() { std::cout.rdbuf(old); }
};

LocalizedRangeScanVector pick(Session* s, const int32_t* idx, int n) {
  LocalizedRangeScanVector v;
  for (int i = 0; i < n; i++) v.push_back(s->scans.at(idx[i]));
  return v;
}

// MatchScan steps 1-4 + AddScans (Mapper.cpp:195-225) without the sweeps
void position_grid_and_add(Session* s, LocalizedRangeScan* scan, const LocalizedRangeScanVector& base) {
  ScanMatcher* m = s->matcher;
  Pose2 scanPose = scan->GetSensorPose();
  Rectangle2<kt_int32s> roi = m->m_pCorrelationGrid->GetROI();
  Vector2<kt_double> offset;
  offset.SetX(scanPose.GetX() - (0.5 * (roi.GetWidth() - 1) * m->m_pCorrelationGrid->GetResolution()));
  offset.SetY(scanPose.GetY() - (0.5 * (roi.GetHeight() - 1) * m->m_pCorrelationGrid->GetResolution()));
  m->m_pCorrelationGrid->GetCoordinateConverter()->SetOffset(offset);
  m->AddScans(base, scanPose.GetPosition());
}

}  // namespace

extern "C" {

void* ref_session_create(const ref_matcher_params* p, const ref_laser_params* l) {
  CoutSilencer quiet;
  try {
    Session* s = new Session();
    std::stringstream nm;
    nm << "ref_laser_" << (g_session_counter++);
    s->name = Name(nm.str());
    s->lrf = LaserRangeFinder::CreateLaserRangeFinder(static_cast<LaserRangeFinderType>(l->type), s->name);
    if (l->type == LaserRangeFinder_Custom) {
      s->lrf->SetMinimumRange(l->min_range);
      s->lrf->SetMaximumRange(l->max_range);
      s->lrf->SetMinimumAngle(l->min_angle);
      s->lrf->SetMaximumAngle(l->max_angle);
      s->lrf->SetAngularResolution(l->angular_resolution);
    }
    s->lrf->SetRangeThreshold(l->range_threshold);
    s->lrf->SetOffsetPose(Pose2(l->offset_pose[0], l->offset_pose[1], l->offset_pose[2]));
    SensorManager::GetInstance()->RegisterSensor(s->lrf);

    s->mapper = new Mapper();
    s->mapper->m_pDistanceVariancePenalty->SetValue(p->distance_variance_penalty);
    s->mapper->m_pAngleVariancePenalty->SetValue(p->angle_variance_penalty);
    s->mapper->m_pFineSearchAngleOffset->SetValue(p->fine_search_angle_offset);
    s->mapper->m_pCoarseSearchAngleOffset->SetValue(p->coarse_search_angle_offset);
    s->mapper->m_pCoarseAngleResolution->SetValue(p->coarse_angle_resolution);
    s->mapper->m_pMinimumAnglePenalty->SetValue(p->minimum_angle_penalty);
    s->mapper->m_pMinimumDistancePenalty->SetValue(p->minimum_distance_penalty);
    s->mapper->m_pUseResponseExpansion->SetValue(p->use_response_expansion != 0);

    s->matcher = ScanMatcher::Create(s->mapper, p->search_size, p->resolution, p->smear_deviation,
                                     p->range_threshold);
    if (s->matcher == NULL) {
      SensorManager::GetInstance()->UnregisterSensor(s->lrf);
      delete s->lrf;
      delete s->mapper;
      delete s;
      return NULL;
    }
    return s;
  } catch (...) {
    return NULL;
  }
}

void ref_session_destroy(void* h) {
  CoutSilencer quiet;
  Session* s = static_cast<Session*>(h);
  if (!s) return;
  for (auto* sc : s->scans) delete sc;
  delete s->matcher;
  delete s->mapper;
  SensorManager::GetInstance()->UnregisterSensor(s->lrf);
  delete s->lrf;
  delete s;
}

int ref_n_readings(void* h) { return static_cast<Session*>(h)->lrf->GetNumberOfRangeReadings(); }

// LaserRangeFinder::Validate() recomputes the beam count WITHOUT the +1
// (Karto.h:4152-4161) — Mapper::Process does this to every sensor.
int ref_laser_validate(void* h) {
  CoutSilencer quiet;
  Session* s = static_cast<Session*>(h);
  s->lrf->Validate();
  return s->lrf->GetNumberOfRangeReadings();
}

int ref_scan_add(void* h, const double* ranges, int n, const double pose[3]) {
  Session* s = static_cast<Session*>(h);
  RangeReadingsVector r(ranges, ranges + n);
  LocalizedRangeScan* sc = new LocalizedRangeScan(s->name, r);
  sc->SetOdometricPose(Pose2(pose[0], pose[1], pose[2]));
  sc->SetCorrectedPose(Pose2(pose[0], pose[1], pose[2]));
  s->scans.push_back(sc);
  return static_cast<int>(s->scans.size()) - 1;
}

void ref_scan_set_pose(void* h, int scan, const double pose[3]) {
  Session* s = static_cast<Session*>(h);
  s->scans.at(scan)->SetOdometricPose(Pose2(pose[0], pose[1], pose[2]));
  s->scans.at(scan)->SetCorrectedPose(Pose2(pose[0], pose[1], pose[2]));
}

void ref_scan_sensor_pose(void* h, int scan, double out[3]) {
  Pose2 p = static_cast<Session*>(h)->scans.at(scan)->GetSensorPose();
  out[0] = p.GetX(); out[1] = p.GetY(); out[2] = p.GetHeading();
}

// unfiltered (want_filtered=0) or filtered point readings; returns count
int ref_scan_point_readings(void* h, int scan, int want_filtered, double* out_xy, int cap) {
  const PointVectorDouble& pts = static_cast<Session*>(h)->scans.at(scan)->GetPointReadings(want_filtered != 0);
  int n = static_cast<int>(pts.size());
  for (int i = 0; i < n && i < cap; i++) {
    out_xy[2 * i] = pts[i].GetX();
    out_xy[2 * i + 1] = pts[i].GetY();
  }
  return n;
}

int ref_find_valid_points(void* h, int scan, const double viewpoint[2], double* out_xy, int cap) {
  Session* s = static_cast<Session*>(h);
  PointVectorDouble pts = s->matcher->FindValidPoints(s->scans.at(scan), Vector2<kt_double>(viewpoint[0], viewpoint[1]));
  int n = static_cast<int>(pts.size());
  for (int i = 0; i < n && i < cap; i++) {
    out_xy[2 * i] = pts[i].GetX();
    out_xy[2 * i + 1] = pts[i].GetY();
  }
  return n;
}

// info: width,height,widthStep,dataSize,roi.x,roi.y,roi.w,roi.h,kernelSize ; off: grid offset (m)
void ref_grid_info(void* h, int32_t info[9], double off[2]) {
  CorrelationGrid* g = static_cast<Session*>(h)->matcher->m_pCorrelationGrid;
  info[0] = g->GetWidth(); info[1] = g->GetHeight(); info[2] = g->GetWidthStep(); info[3] = g->GetDataSize();
  info[4] = g->GetROI().GetX(); info[5] = g->GetROI().GetY();
  info[6] = g->GetROI().GetWidth(); info[7] = g->GetROI().GetHeight();
  info[8] = g->m_KernelSize;
  off[0] = g->GetCoordinateConverter()->GetOffset().GetX();
  off[1] = g->GetCoordinateConverter()->GetOffset().GetY();
}

void ref_grid_copy(void* h, uint8_t* out) {
  CorrelationGrid* g = static_cast<Session*>(h)->matcher->m_pCorrelationGrid;
  std::memcpy(out, g->GetDataPointer(), g->GetDataSize());
}

void ref_kernel_copy(void* h, uint8_t* out) {
  CorrelationGrid* g = static_cast<Session*>(h)->matcher->m_pCorrelationGrid;
  std::memcpy(out, g->m_pKernel, g->m_KernelSize * g->m_KernelSize);
}

int ref_set_grid_from_scans(void* h, int scan, const int32_t* base, int nbase) {
  Session* s = static_cast<Session*>(h);
  try {
    position_grid_and_add(s, s->scans.at(scan), pick(s, base, nbase));
    return 0;
  } catch (...) {
    return -1;
  }
}

// returns status (0 ok, -2 exception); *response gets the return value
int ref_match_scan(void* h, int scan, const int32_t* base, int nbase, int do_penalize, int do_refine,
                   double* response, double mean[3], double cov[9]) {
  Session* s = static_cast<Session*>(h);
  try {
    Pose2 m;
    Matrix3 c;
    *response = s->matcher->MatchScan(s->scans.at(scan), pick(s, base, nbase), m, c, do_penalize != 0, do_refine != 0);
    mean[0] = m.GetX(); mean[1] = m.GetY(); mean[2] = m.GetHeading();
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) cov[3 * i + j] = c(i, j);
    return 0;
  } catch (...) {
    return -2;
  }
}

// cov is IN/OUT: the fine stage only overwrites cov(2,2) (Mapper.cpp:648,691)
int ref_correlate_scan(void* h, int scan, const double center[3], double off_x, double off_y, double res_x,
                       double res_y, double off_a, double res_a, int do_penalize, int fine, double* response,
                       double mean[3], double cov[9]) {
  Session* s = static_cast<Session*>(h);
  try {
    Pose2 m;
    Matrix3 c;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) c(i, j) = cov[3 * i + j];
    *response = s->matcher->CorrelateScan(s->scans.at(scan), Pose2(center[0], center[1], center[2]),
                                          Vector2<kt_double>(off_x, off_y), Vector2<kt_double>(res_x, res_y), off_a,
                                          res_a, do_penalize != 0, m, c, fine != 0);
    mean[0] = m.GetX(); mean[1] = m.GetY(); mean[2] = m.GetHeading();
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) cov[3 * i + j] = c(i, j);
    return 0;
  } catch (...) {
    return -2;
  }
}

// GridIndexLookup::ComputeOffsets (Karto.h:6409) then copy the tables: out[k*N+i]
int ref_compute_offsets(void* h, int scan, double angle_center, double angle_offset, double angle_res, int32_t* out,
                        int cap) {
  Session* s = static_cast<Session*>(h);
  s->matcher->m_pGridLookup->ComputeOffsets(s->scans.at(scan), angle_center, angle_offset, angle_res);
  int n_angles = static_cast<int>(math::Round(angle_offset * 2.0 / angle_res) + 1);
  int written = 0;
  for (int k = 0; k < n_angles; k++) {
    const LookupArray* a = s->matcher->m_pGridLookup->GetLookupArray(k);
    int n = a->GetSize();
    for (int i = 0; i < n; i++, written++)
      if (written < cap) out[written] = a->GetArrayPointer()[i];
  }
  return n_angles;
}

// the (y, x, theta)-ordered sweep of CorrelateScan (Mapper.cpp:373-424) but
// returning the raw integer numerator of GetResponse: round(resp * N * 100).
// dims[3] = nY, nX, nAngles.  Must be preceded by ref_set_grid_from_scans / ref_match_scan.
int ref_response_sums(void* h, int scan, const double center[3], double off_x, double off_y, double res_x,
                      double res_y, double off_a, double res_a, int32_t* out, int cap, int32_t dims[3]) {
  Session* s = static_cast<Session*>(h);
  ScanMatcher* m = s->matcher;
  try {
    m->m_pGridLookup->ComputeOffsets(s->scans.at(scan), center[2], off_a, res_a);
    int nX = static_cast<int>(math::Round(off_x * 2.0 / res_x) + 1);
    int nY = static_cast<int>(math::Round(off_y * 2.0 / res_y) + 1);
    int nA = static_cast<int>(math::Round(off_a * 2.0 / res_a) + 1);
    dims[0] = nY; dims[1] = nX; dims[2] = nA;
    double n_pts = static_cast<double>(m->m_pGridLookup->GetLookupArray(0)->GetSize());
    int w = 0;
    for (int iy = 0; iy < nY; iy++) {
      double newY = center[1] + (-off_y + iy * res_y);
      for (int ix = 0; ix < nX; ix++) {
        double newX = center[0] + (-off_x + ix * res_x);
        Vector2<kt_int32s> gp = m->m_pCorrelationGrid->WorldToGrid(Vector2<kt_double>(newX, newY));
        kt_int32s gi = m->m_pCorrelationGrid->GridIndex(gp);
        for (int k = 0; k < nA; k++, w++) {
          double r = m->GetResponse(k, gi);
          if (w < cap) out[w] = static_cast<int32_t>(std::llround(r * n_pts * 100.0));
        }
      }
    }
    return 0;
  } catch (...) {
    return -2;
  }
}

// median-free raw timing helper: runs CorrelateScan `reps` times, returns seconds per call (min over reps)
double ref_time_correlate(void* h, int scan, const double center[3], double off_x, double off_y, double res_x,
                          double res_y, double off_a, double res_a, int do_penalize, int fine, int reps,
                          double* all_secs) {
  Session* s = static_cast<Session*>(h);
  double best = 1e30;
  for (int r = 0; r < reps; r++) {
    Pose2 m;
    Matrix3 c;
    auto t0 = std::chrono::steady_clock::now();
    s->matcher->CorrelateScan(s->scans.at(scan), Pose2(center[0], center[1], center[2]),
                              Vector2<kt_double>(off_x, off_y), Vector2<kt_double>(res_x, res_y), off_a, res_a,
                              do_penalize != 0, m, c, fine != 0);
    auto t1 = std::chrono::steady_clock::now();
    double sec = std::chrono::duration<double>(t1 - t0).count();
    if (all_secs) all_secs[r] = sec;
    best = std::min(best, sec);
  }
  return best;
}

double ref_time_match_scan(void* h, int scan, const int32_t* base, int nbase, int reps, double* all_secs) {
  Session* s = static_cast<Session*>(h);
  double best = 1e30;
  LocalizedRangeScanVector b = pick(s, base, nbase);
  for (int r = 0; r < reps; r++) {
    Pose2 m;
    Matrix3 c;
    auto t0 = std::chrono::steady_clock::now();
    s->matcher->MatchScan(s->scans.at(scan), b, m, c, true, true);
    auto t1 = std::chrono::steady_clock::now();
    double sec = std::chrono::duration<double>(t1 - t0).count();
    if (all_secs) all_secs[r] = sec;
    best = std::min(best, sec);
  }
  return best;
}

// ---------------- karto::OccupancyGrid (Karto.h:5609-6039) ----------------

void* ref_occgrid_create(void* h, const int32_t* scans, int n, double resolution, int32_t dims[3], double off[2]) {
  Session* s = static_cast<Session*>(h);
  try {
    OccupancyGrid* g = OccupancyGrid::CreateFromScans(pick(s, scans, n), resolution);
    if (!g) return NULL;
    dims[0] = g->GetWidth(); dims[1] = g->GetHeight(); dims[2] = g->GetWidthStep();
    off[0] = g->GetCoordinateConverter()->GetOffset().GetX();
    off[1] = g->GetCoordinateConverter()->GetOffset().GetY();
    return g;
  } catch (...) {
    return NULL;
  }
}

void ref_occgrid_copy(void* g_, uint8_t* cells, uint32_t* pass, uint32_t* hit) {
  OccupancyGrid* g = static_cast<OccupancyGrid*>(g_);
  int n = g->GetDataSize();
  if (cells) std::memcpy(cells, g->GetDataPointer(), n);
  if (pass) std::memcpy(pass, g->m_pCellPassCnt->GetDataPointer(), sizeof(uint32_t) * n);
  if (hit) std::memcpy(hit, g->m_pCellHitsCnt->GetDataPointer(), sizeof(uint32_t) * n);
}

void ref_occgrid_destroy(void* g_) { delete static_cast<OccupancyGrid*>(g_); }

double ref_time_occgrid(void* h, const int32_t* scans, int n, double resolution, int reps, double* all_secs) {
  Session* s = static_cast<Session*>(h);
  LocalizedRangeScanVector v = pick(s, scans, n);
  double best = 1e30;
  for (int r = 0; r < reps; r++) {
    auto t0 = std::chrono::steady_clock::now();
    OccupancyGrid* g = OccupancyGrid::CreateFromScans(v, resolution);
    auto t1 = std::chrono::steady_clock::now();
    delete g;
    double sec = std::chrono::duration<double>(t1 - t0).count();
    if (all_secs) all_secs[r] = sec;
    best = std::min(best, sec);
  }
  return best;
}

// Grid<T>::TraceLine cell list (Karto.h:4680-4745) on a w x h grid
int ref_trace_line(int w, int hgt, int x0, int y0, int x1, int y1, int32_t* out_xy, int cap) {
  struct Rec : Functor {
    Grid<kt_int32u>* g; std::vector<int>* v;
    void operator()(kt_int32u index) override {
      Vector2<kt_int32s> p = g->IndexToGrid(index);
      v->push_back(p.GetX()); v->push_back(p.GetY());
    }
  };
  Grid<kt_int32u>* g = Grid<kt_int32u>::CreateGrid(w, hgt, 1.0);
  std::vector<int> v;
  Rec rec; rec.g = g; rec.v = &v;
  g->TraceLine(x0, y0, x1, y1, &rec);
  int n = static_cast<int>(v.size() / 2);
  for (int i = 0; i < n && i < cap; i++) { out_xy[2 * i] = v[2 * i]; out_xy[2 * i + 1] = v[2 * i + 1]; }
  delete g;
  return n;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------
// The whole lesson6 front end: karto::Mapper::Process (Mapper.cpp:1999-2079) on a stream of scans, with the
// reference's own MapperGraph / ScanManager / ScanMatchers.  The struct mirrors b2s_mapper_params (include/b200slam.h);
// values are the ones STORED in the Mapper.  A ScanSolver can be plugged in as four C callbacks (the reference's own
// plug-in interface, Mapper.h:825-891), which lets tests give both sides the same back end.
extern "C" {

struct ref_mapper_params {
  int32_t use_scan_matching, use_scan_barycenter;
  double minimum_time_interval, minimum_travel_distance, minimum_travel_heading;
  int32_t scan_buffer_size, do_loop_closing;
  double scan_buffer_maximum_scan_distance, link_match_minimum_response_fine, link_scan_maximum_distance,
      loop_search_maximum_distance;
  int32_t loop_match_minimum_chain_size, reserved;
  double loop_match_maximum_variance_coarse, loop_match_minimum_response_coarse, loop_match_minimum_response_fine;
  ref_matcher_params sequential, loop;
};

struct ref_scan_solver {
  void* user;
  void (*add_node)(void*, int32_t, const double*);
  void (*add_constraint)(void*, int32_t, int32_t, const double*, const double*);
  int32_t (*compute)(void*, int32_t, int32_t*, double*);
  void (*clear)(void*);
};

}  // extern "C"

namespace {

struct CallbackSolver : ScanSolver {
  ref_scan_solver cb;
  IdPoseVector corrections;
  int n_nodes = 0;
  void Compute() override {
    corrections.clear();
    std::vector<int32_t> ids(n_nodes);
    std::vector<double> poses(3 * static_cast<size_t>(n_nodes));
    int n = cb.compute(cb.user, n_nodes, ids.data(), poses.data());
    for (int i = 0; i < n; i++) corrections.push_back(std::make_pair(ids[i], Pose2(poses[3 * i], poses[3 * i + 1], poses[3 * i + 2])));
  }
  const IdPoseVector& GetCorrections() const override { return corrections; }
  void AddNode(Vertex<LocalizedRangeScan>* v) override {
    Pose2 p = v->GetObject()->GetCorrectedPose();  // as lesson6/src/spa_solver/spa_solver.cc:65-70
    double c[3] = {p.GetX(), p.GetY(), p.GetHeading()};
    n_nodes++;
    cb.add_node(cb.user, v->GetObject()->GetUniqueId(), c);
  }
  void AddConstraint(Edge<LocalizedRangeScan>* e) override {  // as spa_solver.cc:72-93 (pose difference + covariance)
    LinkInfo* li = (LinkInfo*)(e->GetLabel());
    Pose2 d = li->GetPoseDifference();
    double diff[3] = {d.GetX(), d.GetY(), d.GetHeading()}, cov[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) cov[3 * i + j] = li->GetCovariance()(i, j);
    cb.add_constraint(cb.user, e->GetSource()->GetObject()->GetUniqueId(), e->GetTarget()->GetObject()->GetUniqueId(), diff, cov);
  }
  void Clear() override {
    corrections.clear();
    if (cb.clear) cb.clear(cb.user);
  }
};

struct MapperSession {
  Mapper* mapper = nullptr;
  LaserRangeFinder* lrf = nullptr;
  CallbackSolver* solver = nullptr;
  Name name;
  std::vector<LocalizedRangeScan*> all;  // every scan handed to Process (rejected ones too), for deletion
  std::vector<LaserRangeFinder*> extra;  // further sensors (other robots) with the same parameters, ref_mapper_add_sensor
  std::vector<Name> extra_names;
  ref_laser_params lp;
};

LaserRangeFinder* make_lrf(const ref_laser_params* l, const Name& name) {
  LaserRangeFinder* lrf = LaserRangeFinder::CreateLaserRangeFinder(static_cast<LaserRangeFinderType>(l->type), name);
  if (l->type == LaserRangeFinder_Custom) {
    lrf->SetMinimumRange(l->min_range);
    lrf->SetMaximumRange(l->max_range);
    lrf->SetMinimumAngle(l->min_angle);
    lrf->SetMaximumAngle(l->max_angle);
    lrf->SetAngularResolution(l->angular_resolution);
  }
  lrf->SetRangeThreshold(l->range_threshold);
  lrf->SetOffsetPose(Pose2(l->offset_pose[0], l->offset_pose[1], l->offset_pose[2]));
  SensorManager::GetInstance()->RegisterSensor(lrf);
  return lrf;
}

int process_named(MapperSession* s, const Name& name, const double* ranges, int n, const double* odom, double time,
                  double* out_corrected) {
  std::vector<kt_double> r(ranges, ranges + n);
  LocalizedRangeScan* scan = new LocalizedRangeScan(name, r);
  scan->SetOdometricPose(Pose2(odom[0], odom[1], odom[2]));
  scan->SetCorrectedPose(Pose2(odom[0], odom[1], odom[2]));
  scan->SetTime(time);
  s->all.push_back(scan);
  bool ok = s->mapper->Process(scan);
  Pose2 c = scan->GetCorrectedPose();
  if (out_corrected) { out_corrected[0] = c.GetX(); out_corrected[1] = c.GetY(); out_corrected[2] = c.GetHeading(); }
  return ok ? 1 : 0;
}

}  // namespace

extern "C" {

void* ref_mapper_create(const ref_mapper_params* p, const ref_laser_params* l) {
  CoutSilencer quiet;
  MapperSession* s = new MapperSession();
  std::stringstream nm;
  nm << "ref_mapper_laser_" << (g_session_counter++);
  s->name = Name(nm.str());
  s->lp = *l;
  s->lrf = make_lrf(l, s->name);
  Mapper* m = s->mapper = new Mapper();
  m->m_pUseScanMatching->SetValue(p->use_scan_matching != 0);
  m->m_pUseScanBarycenter->SetValue(p->use_scan_barycenter != 0);
  m->m_pMinimumTimeInterval->SetValue(p->minimum_time_interval);
  m->m_pMinimumTravelDistance->SetValue(p->minimum_travel_distance);
  m->m_pMinimumTravelHeading->SetValue(p->minimum_travel_heading);
  m->m_pScanBufferSize->SetValue(p->scan_buffer_size);
  m->m_pScanBufferMaximumScanDistance->SetValue(p->scan_buffer_maximum_scan_distance);
  m->m_pLinkMatchMinimumResponseFine->SetValue(p->link_match_minimum_response_fine);
  m->m_pLinkScanMaximumDistance->SetValue(p->link_scan_maximum_distance);
  m->m_pLoopSearchMaximumDistance->SetValue(p->loop_search_maximum_distance);
  m->m_pDoLoopClosing->SetValue(p->do_loop_closing != 0);
  m->m_pLoopMatchMinimumChainSize->SetValue(p->loop_match_minimum_chain_size);
  m->m_pLoopMatchMaximumVarianceCoarse->SetValue(p->loop_match_maximum_variance_coarse);
  m->m_pLoopMatchMinimumResponseCoarse->SetValue(p->loop_match_minimum_response_coarse);
  m->m_pLoopMatchMinimumResponseFine->SetValue(p->loop_match_minimum_response_fine);
  m->m_pCorrelationSearchSpaceDimension->SetValue(p->sequential.search_size);
  m->m_pCorrelationSearchSpaceResolution->SetValue(p->sequential.resolution);
  m->m_pCorrelationSearchSpaceSmearDeviation->SetValue(p->sequential.smear_deviation);
  m->m_pLoopSearchSpaceDimension->SetValue(p->loop.search_size);
  m->m_pLoopSearchSpaceResolution->SetValue(p->loop.resolution);
  m->m_pLoopSearchSpaceSmearDeviation->SetValue(p->loop.smear_deviation);
  m->m_pDistanceVariancePenalty->SetValue(p->sequential.distance_variance_penalty);
  m->m_pAngleVariancePenalty->SetValue(p->sequential.angle_variance_penalty);
  m->m_pFineSearchAngleOffset->SetValue(p->sequential.fine_search_angle_offset);
  m->m_pCoarseSearchAngleOffset->SetValue(p->sequential.coarse_search_angle_offset);
  m->m_pCoarseAngleResolution->SetValue(p->sequential.coarse_angle_resolution);
  m->m_pMinimumAnglePenalty->SetValue(p->sequential.minimum_angle_penalty);
  m->m_pMinimumDistancePenalty->SetValue(p->sequential.minimum_distance_penalty);
  m->m_pUseResponseExpansion->SetValue(p->sequential.use_response_expansion != 0);
  return s;
}

void ref_mapper_set_solver(void* h, const ref_scan_solver* cb) {
  MapperSession* s = static_cast<MapperSession*>(h);
  s->solver = new CallbackSolver();
  s->solver->cb = *cb;
  s->mapper->SetScanSolver(s->solver);
}

void ref_mapper_destroy(void* h) {
  CoutSilencer quiet;
  MapperSession* s = static_cast<MapperSession*>(h);
  if (!s) return;
  delete s->mapper;
  for (auto* p : s->all) delete p;
  delete s->solver;
  SensorManager::GetInstance()->UnregisterSensor(s->lrf);
  delete s->lrf;
  for (auto* p : s->extra) {
    SensorManager::GetInstance()->UnregisterSensor(p);
    delete p;
  }
  delete s;
}

// what karto_slam.cc:437-475 does per LaserScan: build the LocalizedRangeScan, set both poses from odometry, Process
int ref_mapper_scan_count(void* h);

int ref_mapper_process(void* h, const double* ranges, int n, const double* odom, double time, double* out_corrected) {
  CoutSilencer quiet;
  MapperSession* s = static_cast<MapperSession*>(h);
  return process_named(s, s->name, ranges, n, odom, time, out_corrected);
}

// a further sensor (another robot's laser, same parameters).  `prefix` decides where its name sorts relative to the
// session's own "ref_mapper_laser_<n>" (Name::operator< compares strings, Karto.h:484).  Returns its index (>= 1).
int ref_mapper_add_sensor(void* h, const char* prefix) {
  CoutSilencer quiet;
  MapperSession* s = static_cast<MapperSession*>(h);
  std::stringstream nm;
  nm << prefix << "_" << (g_session_counter++);
  Name name(nm.str());
  s->extra.push_back(make_lrf(&s->lp, name));
  s->extra_names.push_back(name);
  return static_cast<int>(s->extra.size());
}

// sensor 0 = the session's own laser, k >= 1 = the k-th added one
int ref_mapper_process_sensor(void* h, int sensor, const double* ranges, int n, const double* odom, double time,
                              double* out_corrected) {
  CoutSilencer quiet;
  MapperSession* s = static_cast<MapperSession*>(h);
  return process_named(s, sensor == 0 ? s->name : s->extra_names[sensor - 1], ranges, n, odom, time, out_corrected);
}

// corrected poses in unique-id order (MapperSensorManager::GetScan(id), Mapper.h:1486-1498); GetAllProcessedScans is
// sensor-major
void ref_mapper_get_poses_by_id(void* h, double* out) {
  MapperSession* s = static_cast<MapperSession*>(h);
  const int n = ref_mapper_scan_count(h);
  for (int i = 0; i < n; i++) {
    Pose2 c = s->mapper->m_pMapperSensorManager->GetScan(i)->GetCorrectedPose();
    out[3 * i] = c.GetX(); out[3 * i + 1] = c.GetY(); out[3 * i + 2] = c.GetHeading();
  }
}

int ref_mapper_scan_count(void* h) {
  MapperSession* s = static_cast<MapperSession*>(h);
  return s->mapper->m_Initialized ? static_cast<int>(s->mapper->GetAllProcessedScans().size()) : 0;
}

void ref_mapper_get_poses(void* h, double* out) {
  MapperSession* s = static_cast<MapperSession*>(h);
  LocalizedRangeScanVector v = s->mapper->GetAllProcessedScans();
  for (size_t i = 0; i < v.size(); i++) {
    Pose2 c = v[i]->GetCorrectedPose();
    out[3 * i] = c.GetX(); out[3 * i + 1] = c.GetY(); out[3 * i + 2] = c.GetHeading();
  }
}

int ref_mapper_edge_count(void* h) {
  MapperSession* s = static_cast<MapperSession*>(h);
  return s->mapper->m_Initialized ? static_cast<int>(s->mapper->GetGraph()->GetEdges().size()) : 0;
}

void ref_mapper_get_edges(void* h, int32_t* ids, double* diff, double* cov) {
  MapperSession* s = static_cast<MapperSession*>(h);
  const std::vector<Edge<LocalizedRangeScan>*>& e = s->mapper->GetGraph()->GetEdges();
  for (size_t i = 0; i < e.size(); i++) {
    LinkInfo* li = (LinkInfo*)(e[i]->GetLabel());
    ids[2 * i] = e[i]->GetSource()->GetObject()->GetUniqueId();
    ids[2 * i + 1] = e[i]->GetTarget()->GetObject()->GetUniqueId();
    Pose2 d = li->GetPoseDifference();
    diff[3 * i] = d.GetX(); diff[3 * i + 1] = d.GetY(); diff[3 * i + 2] = d.GetHeading();
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) cov[9 * i + 3 * r + c] = li->GetCovariance()(r, c);
  }
}

// Mapper::InitializeParameters (Mapper.cpp:1448-1653): the defaults as a fresh reference Mapper holds them
void ref_mapper_default_params(ref_mapper_params* p) {
  CoutSilencer quiet;
  Mapper m;
  std::memset(p, 0, sizeof(*p));
  p->use_scan_matching = m.m_pUseScanMatching->GetValue();
  p->use_scan_barycenter = m.m_pUseScanBarycenter->GetValue();
  p->minimum_time_interval = m.m_pMinimumTimeInterval->GetValue();
  p->minimum_travel_distance = m.m_pMinimumTravelDistance->GetValue();
  p->minimum_travel_heading = m.m_pMinimumTravelHeading->GetValue();
  p->scan_buffer_size = m.m_pScanBufferSize->GetValue();
  p->do_loop_closing = m.m_pDoLoopClosing->GetValue();
  p->scan_buffer_maximum_scan_distance = m.m_pScanBufferMaximumScanDistance->GetValue();
  p->link_match_minimum_response_fine = m.m_pLinkMatchMinimumResponseFine->GetValue();
  p->link_scan_maximum_distance = m.m_pLinkScanMaximumDistance->GetValue();
  p->loop_search_maximum_distance = m.m_pLoopSearchMaximumDistance->GetValue();
  p->loop_match_minimum_chain_size = m.m_pLoopMatchMinimumChainSize->GetValue();
  p->loop_match_maximum_variance_coarse = m.m_pLoopMatchMaximumVarianceCoarse->GetValue();
  p->loop_match_minimum_response_coarse = m.m_pLoopMatchMinimumResponseCoarse->GetValue();
  p->loop_match_minimum_response_fine = m.m_pLoopMatchMinimumResponseFine->GetValue();
  ref_matcher_params t;
  std::memset(&t, 0, sizeof(t));
  t.distance_variance_penalty = m.m_pDistanceVariancePenalty->GetValue();
  t.angle_variance_penalty = m.m_pAngleVariancePenalty->GetValue();
  t.fine_search_angle_offset = m.m_pFineSearchAngleOffset->GetValue();
  t.coarse_search_angle_offset = m.m_pCoarseSearchAngleOffset->GetValue();
  t.coarse_angle_resolution = m.m_pCoarseAngleResolution->GetValue();
  t.minimum_angle_penalty = m.m_pMinimumAnglePenalty->GetValue();
  t.minimum_distance_penalty = m.m_pMinimumDistancePenalty->GetValue();
  t.use_response_expansion = m.m_pUseResponseExpansion->GetValue();
  p->sequential = t;
  p->sequential.search_size = m.m_pCorrelationSearchSpaceDimension->GetValue();
  p->sequential.resolution = m.m_pCorrelationSearchSpaceResolution->GetValue();
  p->sequential.smear_deviation = m.m_pCorrelationSearchSpaceSmearDeviation->GetValue();
  p->loop = t;
  p->loop.search_size = m.m_pLoopSearchSpaceDimension->GetValue();
  p->loop.resolution = m.m_pLoopSearchSpaceResolution->GetValue();
  p->loop.smear_deviation = m.m_pLoopSearchSpaceSmearDeviation->GetValue();
}

int ref_mapper_running_count(void* h) {
  MapperSession* s = static_cast<MapperSession*>(h);
  return static_cast<int>(s->mapper->m_pMapperSensorManager->GetRunningScans(s->name).size());
}

}  // extern "C"
