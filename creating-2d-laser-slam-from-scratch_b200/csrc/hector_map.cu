// K2a + K3 — lesson4 Hector log-odds grid map update and Gauss-Newton scan-to-map alignment on H100 (sm_90a).
// Product code: CUDA only.
//
// Reference behaviour (paths relative to reference/lesson4/include/lesson4/hector_mapping):
//   OccGridMapBase::updateByScan / updateLineBresenhami / bresenham2D / bresenhamCellFree/Occ   map/OccGridMapBase.h:118-168, 220-330
//   LogOddsCell, GridMapLogOddsFunctions                                                       map/GridMapLogOdds.h:37-161
//   GridMapBase ctor, setMapTransformation, getMapCoordsPose, getWorldCoordsPose               map/GridMapBase.h:54-66, 229-286
//   OccGridMapUtil::getCompleteHessianDerivs / interpMapValueWithDerivatives                   map/OccGridMapUtil.h:77-228
//   ScanMatcher::matchData / estimateTransformationLogLh                                       matcher/ScanMatcher.h:60-141
//
// K2a is sequential ACROSS scans (the <50 clamp and the once-per-scan stamps) but parallel WITHIN a scan.  The
// reference's in-scan order dependence is reproduced exactly with two passes over the rays (one warp per beam,
// closed-form Bresenham: minor-axis steps after n major steps = floor((da/2 + n*db) / da)):
//   mark  : every traversed cell records the LOWEST beam index that frees it / ends on it (64-bit atomicMax of
//           (scan epoch << 32 | ~beam));
//   apply : the recorded winner beam applies the cell's update once: free-only cells get += logOddsFree; end cells
//           get the reference's "(v + f) - f" un-free rounding iff a lower-indexed beam had freed them first, then
//           += logOddsOccupied if v < 50 — identical floats to the sequential loop, whatever the execution order.
// The pose's cosf/sinf are taken on the host (glibc) so that all device arithmetic on the integer path is + - *
// in float32 without FMA: the truncated cell coordinates are bit-identical to the CPU.
// K3 runs the whole 1 + maxIterations Gauss-Newton loop of one grid level in ONE kernel launch: per-point terms in
// parallel, then thread 0 accumulates H and dTr in point order (the reference's float32 summation order).
//
// HBM layout per cell: logOdds f32, updateIndex i32 (the reference's LogOddsCell, split SoA), + two u64 stamps.
//
// Shared with the processor (hector_slam.cu) through hector_grid.cuh: the map transform, the begin / end cells, the
// Bresenham set-up and step, the bilinear bounds test and finish, the 3x3 solve, normalize_angle and the ROS map.
// This handle's own: 64-bit stamps and a per-beam apply pass, the begin cell on the host, the updateByScanJustOnce end
// cell, probabilities through the float expf and log-odds factors through logf.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "hector_grid.cuh"

using namespace b2s;

struct b2s_hector_map {
  Stream stream;
  int device = 0;
  int sx = 0, sy = 0;
  MapTransform tf = {};
  float lo_free = 0, lo_occ = 0;
  int curr_update_index = 0;
  unsigned int epoch = 0;
  Buf<float> d_lo;
  Buf<int32_t> d_ui;
  Buf<unsigned long long> d_free, d_occ;
  Buf<float> d_pts;
  Buf<float> d_out;  // [3 pose + 9 H]
  Buf<unsigned long long> d_visits;
  double last_ms[2] = {0, 0};
  Event ev[4];  // update begin/end, match begin/end
};

namespace b2s {

// end cell + updateLineBresenhami set-up
__device__ __forceinline__ BresenhamLine hc_line(float c, float s, float mx, float my, bool just_once, int bx, int by,
                                                 float px, float py, int sx, int sy) {
  const int2 end = just_once ? just_once_end_cell(bx, by, px, py) : end_cell(c, s, mx, my, px, py);
  return bresenham_line(bx, by, end, sx, sy);
}

// pass 1: record, per traversed cell, the lowest beam index that frees it / ends on it
__global__ void __launch_bounds__(256)
    k_hc_mark(const float *__restrict__ pts, int n, float c, float s, float mx, float my, bool just_once, int bx, int by, int sx, int sy,
              unsigned long long epoch_hi, unsigned long long *__restrict__ free_st,
              unsigned long long *__restrict__ occ_st) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = warp0; i < n; i += nwarps) {
    const BresenhamLine L = hc_line(c, s, mx, my, just_once, bx, by, pts[2 * i], pts[2 * i + 1], sx, sy);
    if (!L.ok) continue;
    const unsigned long long stamp = epoch_hi | (unsigned long long)(0xffffffffu - (unsigned int)i);
    const int start = L.y0 * sx + L.x0;
    for (unsigned int k = lane; k < L.da; k += 32) atomicMax(free_st + bresenham_offset(L, start, k), stamp);
    if (lane == 0) atomicMax(occ_st + (L.y1 * sx + L.x1), stamp);
  }
}

// pass 2: the winner beam of each cell applies the reference's update exactly once
__global__ void __launch_bounds__(256)
    k_hc_apply(const float *__restrict__ pts, int n, float c, float s, float mx, float my, bool just_once, int bx, int by, int sx, int sy,
               unsigned long long epoch_hi, const unsigned long long *__restrict__ free_st,
               const unsigned long long *__restrict__ occ_st, float lo_free, float lo_occ, int mark_free, int mark_occ,
               float *__restrict__ lo, int32_t *__restrict__ ui, unsigned long long *__restrict__ visits) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long my_visits = 0;
  for (int i = warp0; i < n; i += nwarps) {
    const BresenhamLine L = hc_line(c, s, mx, my, just_once, bx, by, pts[2 * i], pts[2 * i + 1], sx, sy);
    if (!L.ok) continue;
    const unsigned long long stamp = epoch_hi | (unsigned long long)(0xffffffffu - (unsigned int)i);
    const int start = L.y0 * sx + L.x0;
    for (unsigned int k = lane; k < L.da; k += 32) {
      const int off = bresenham_offset(L, start, k);
      my_visits++;
      if (free_st[off] == stamp && (occ_st[off] >> 32) != (epoch_hi >> 32)) {
        // freed this scan, never an end point: bresenhamCellFree (OccGridMapBase.h:302-312)
        lo[off] = __fadd_rn(lo[off], lo_free);
        ui[off] = mark_free;
      }
    }
    if (lane == 0) {
      my_visits++;
      const int off = L.y1 * sx + L.x1;
      if (occ_st[off] == stamp) {  // bresenhamCellOcc (OccGridMapBase.h:315-330), first beam ending here
        float v = lo[off];
        const unsigned long long fs = free_st[off];
        if ((fs >> 32) == (epoch_hi >> 32) && fs > stamp) {  // a LOWER beam index freed it first: set free, then unset
          v = __fadd_rn(v, lo_free);
          v = __fsub_rn(v, lo_free);
        }
        if (v < 50.0f) v = __fadd_rn(v, lo_occ);
        lo[off] = v;
        ui[off] = mark_occ;
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) my_visits += __shfl_xor_sync(0xffffffffu, my_visits, d);
  if (lane == 0 && my_visits) atomicAdd(visits, my_visits);
}

// ---- K3: Gauss-Newton scan-to-map alignment (one grid level), whole iteration loop in one launch ----

// getGridProbability (GridMapLogOdds.h:136-140) with the device's float expf, where the reference rounds the C library's
// double exp to float (as the processor's log_odds_prob does): the values can differ in the last bits, which is why
// b2s_hector_map_match_data is held to 1e-4 of the reference rather than bit for bit.
__device__ __forceinline__ float hc_prob(const float *__restrict__ lo, int index) {
  const float odds = expf(lo[index]);
  return odds / (odds + 1.0f);
}

__device__ __forceinline__ void hc_interp(const float *__restrict__ lo, int sx, int sy, float x, float y, float out[3]) {
  if (!interp_inside(sx, sy, x, y)) { out[0] = out[1] = out[2] = 0.0f; return; }
  const int ix = (int)x, iy = (int)y;
  const int index = iy * sx + ix;
  interp_finish(hc_prob(lo, index), hc_prob(lo, index + 1), hc_prob(lo, index + sx), hc_prob(lo, index + sx + 1),
                x - (float)ix, y - (float)iy, out);
}

constexpr int GN_THREADS = 512;
constexpr int GN_CHUNK = 1024;  // points staged per pass

__global__ void __launch_bounds__(GN_THREADS)
    k_hc_match(const float *__restrict__ lo, int sx, int sy, const float *__restrict__ pts, int n, float e0, float e1,
               float e2, int iterations, MapTransform tf, float *__restrict__ out) {
  __shared__ float terms[GN_CHUNK][4];  // t1, t2, rotDeriv, funVal per point
  __shared__ float est[3];
  __shared__ float H[9], dTr[3];
  if (threadIdx.x == 0) { est[0] = e0; est[1] = e1; est[2] = e2; }
  __syncthreads();
  for (int it = 0; it < iterations; it++) {
    const float c = cosf(est[2]), s = sinf(est[2]);
    if (threadIdx.x == 0) {
      for (int q = 0; q < 9; q++) H[q] = 0.0f;
      dTr[0] = dTr[1] = dTr[2] = 0.0f;
    }
    for (int base = 0; base < n; base += GN_CHUNK) {
      const int cnt = min(GN_CHUNK, n - base);
      __syncthreads();
      for (int i = threadIdx.x; i < cnt; i += GN_THREADS) {
        const float px = pts[2 * (base + i)], py = pts[2 * (base + i) + 1];
        const float tx = (c * px + (-s) * py) + est[0], ty = (s * px + c * py) + est[1];
        float t[3];
        hc_interp(lo, sx, sy, tx, ty, t);
        terms[i][0] = t[1];
        terms[i][1] = t[2];
        terms[i][2] = ((-s * px - c * py) * t[1] + (c * px - s * py) * t[2]);
        terms[i][3] = 1.0f - t[0];
      }
      __syncthreads();
      if (threadIdx.x == 0) {  // getCompleteHessianDerivs accumulation, in point order (OccGridMapUtil.h:99-126)
        for (int i = 0; i < cnt; i++) {
          const float t1 = terms[i][0], t2 = terms[i][1], rot = terms[i][2], fun = terms[i][3];
          dTr[0] += t1 * fun;
          dTr[1] += t2 * fun;
          dTr[2] += rot * fun;
          H[0] += t1 * t1;
          H[4] += t2 * t2;
          H[8] += rot * rot;
          H[1] += t1 * t2;
          H[2] += t1 * rot;
          H[5] += t2 * rot;
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      H[3] = H[1]; H[6] = H[2]; H[7] = H[5];
      if (H[0] != 0.0f && H[4] != 0.0f) {  // estimateTransformationLogLh (ScanMatcher.h:107-141)
        float dir[3];
        inv3_mul(H, dTr, dir);
        if (dir[2] > 0.2f) dir[2] = 0.2f;
        else if (dir[2] < -0.2f) dir[2] = -0.2f;
        est[0] += dir[0]; est[1] += dir[1]; est[2] += dir[2];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    get_world_coords(tf, est[0], est[1], out[0], out[1]);
    out[2] = util_normalize_angle(est[2]);
    for (int q = 0; q < 9; q++) out[3 + q] = H[q];
  }
}

}  // namespace b2s

extern "C" void b2s_hector_map_destroy(b2s_hector_map *m);
extern "C" {

b2s_status b2s_hector_map_create(int size_x, int size_y, float resolution, float start_x, float start_y, int device,
                                 void *cuda_stream, b2s_hector_map **out) {
  if (!out || size_x <= 2 || size_y <= 2 || !(resolution > 0.0f)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_map_create: bad size/resolution");
  *out = nullptr;
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<b2s_hector_map, decltype(&b2s_hector_map_destroy)> m(new (std::nothrow) b2s_hector_map(), b2s_hector_map_destroy);
  if (!m) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  m->device = device;
  m->sx = size_x; m->sy = size_y;
  // MapRepMultiMap ctor (MapRepMultiMap.h:63-67): the map's offset
  const float total_x = resolution * (float)size_x, total_y = resolution * (float)size_y;
  m->tf = map_transform(resolution, total_x * start_x, total_y * start_y);
  m->lo_free = prob_to_log_odds_logf(0.4f);
  m->lo_occ = prob_to_log_odds_logf(0.6f);
  B2S_CUDA_CHECK(m->stream.init(cuda_stream));
  for (auto &e : m->ev) B2S_CUDA_CHECK(e.create());
  const size_t cells = (size_t)size_x * size_y;
  B2S_CUDA_CHECK(m->d_lo.reserve(cells));
  B2S_CUDA_CHECK(m->d_ui.reserve(cells));
  B2S_CUDA_CHECK(m->d_free.reserve(cells));
  B2S_CUDA_CHECK(m->d_occ.reserve(cells));
  B2S_CUDA_CHECK(m->d_out.reserve(12));
  B2S_CUDA_CHECK(m->d_visits.reserve(1));
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_lo, 0, cells * 4, m->stream));     // resetGridCell: logOdds 0
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_ui, 0xff, cells * 4, m->stream));  // updateIndex -1
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_free, 0, cells * 8, m->stream));
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_occ, 0, cells * 8, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  m->epoch = 0;
  *out = m.release();
  return B2S_OK;
}

void b2s_hector_map_destroy(b2s_hector_map *m) {
  if (!m) return;
  cudaSetDevice(m->device);
  cudaStreamSynchronize(m->stream);
  delete m;
}

b2s_status b2s_hector_map_set_factors(b2s_hector_map *m, float update_free, float update_occupied) {
  if (!m) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  m->lo_free = prob_to_log_odds_logf(update_free);
  m->lo_occ = prob_to_log_odds_logf(update_occupied);
  return B2S_OK;
}

static b2s_status hc_upload_points(b2s_hector_map *m, const float *points, int n) {
  B2S_CUDA_CHECK(m->d_pts.reserve(2 * (size_t)n));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_pts, points, sizeof(float) * 2 * (size_t)n, cudaMemcpyHostToDevice, m->stream));
  return B2S_OK;
}

static b2s_status hc_update(b2s_hector_map *m, const float *points, int n_points, const float origo[2],
                            const float world_pose[3], bool just_once) {
  B2S_NVTX("K2a updateByScan");
  if (!m || !origo || !world_pose || n_points < 0 || (n_points > 0 && !points)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int mark_free = m->curr_update_index + 1, mark_occ = m->curr_update_index + 2;  // OccGridMapBase.h:120-121
  float mx, my;
  get_map_coords(m->tf, world_pose[0], world_pose[1], mx, my);
  float heading = world_pose[2];
  if (just_once) { mx = 800.0f; my = 800.0f; heading = 0.0f; }  // Eigen::Vector3f mapPose(800, 800, 0) (OccGridMapBase.h:182)
  const float c = cosf(heading), s = sinf(heading);  // Rotation2Df: std::cos / std::sin on float, taken on the host (glibc)
  const int2 b0 = begin_cell(c, s, mx, my, origo[0], origo[1]);
  m->epoch++;
  const unsigned long long epoch_hi = (unsigned long long)m->epoch << 32;
  if (n_points > 0) {
    b2s_status st = hc_upload_points(m, points, n_points);
    if (st) return st;
    B2S_CUDA_CHECK(cudaMemsetAsync(m->d_visits, 0, sizeof(unsigned long long), m->stream));
    const int blocks = std::min(ceil_div(n_points, 8), sm_count(m->device) * 8);
    B2S_CUDA_CHECK(cudaEventRecord(m->ev[0], m->stream));
    k_hc_mark<<<blocks, 256, 0, m->stream>>>(m->d_pts, n_points, c, s, mx, my, just_once, b0.x, b0.y, m->sx, m->sy, epoch_hi,
                                             m->d_free, m->d_occ);
    k_hc_apply<<<blocks, 256, 0, m->stream>>>(m->d_pts, n_points, c, s, mx, my, just_once, b0.x, b0.y, m->sx, m->sy, epoch_hi,
                                              m->d_free, m->d_occ,
                                              m->lo_free, m->lo_occ, mark_free, mark_occ, m->d_lo, m->d_ui, m->d_visits);
    B2S_CUDA_CHECK(cudaEventRecord(m->ev[1], m->stream));
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  m->curr_update_index += 3;  // OccGridMapBase.h:167
  return B2S_OK;
}

b2s_status b2s_hector_map_update_by_scan(b2s_hector_map *m, const float *points, int n_points, const float origo[2],
                                         const float world_pose[3]) {
  return hc_update(m, points, n_points, origo, world_pose, false);
}

b2s_status b2s_hector_map_update_by_scan_just_once(b2s_hector_map *m, const float *points, int n_points,
                                                   const float origo[2]) {
  const float unused_pose[3] = {0.0f, 0.0f, 0.0f};
  return hc_update(m, points, n_points, origo, unused_pose, true);
}

b2s_status b2s_hector_map_match_data(b2s_hector_map *m, const float *points, int n_points,
                                     const float begin_world_pose[3], int max_iterations, float out_world_pose[3],
                                     float out_cov[9]) {
  if (!m || !begin_world_pose || !out_world_pose || !out_cov || n_points < 0 || max_iterations < 0 || (n_points > 0 && !points))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (n_points == 0) {  // ScanMatcher.h:66,97: no data -> begin estimate returned unchanged
    std::memcpy(out_world_pose, begin_world_pose, 3 * sizeof(float));
    return B2S_OK;
  }
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  b2s_status st = hc_upload_points(m, points, n_points);
  if (st) return st;
  float e0, e1;
  get_map_coords(m->tf, begin_world_pose[0], begin_world_pose[1], e0, e1);
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[2], m->stream));
  k_hc_match<<<1, GN_THREADS, 0, m->stream>>>(m->d_lo, m->sx, m->sy, m->d_pts, n_points, e0, e1, begin_world_pose[2],
                                              1 + max_iterations, m->tf, m->d_out);
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[3], m->stream));
  B2S_CUDA_CHECK(cudaGetLastError());
  float host[12];
  B2S_CUDA_CHECK(cudaMemcpyAsync(host, m->d_out, sizeof(host), cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  std::memcpy(out_world_pose, host, 3 * sizeof(float));
  std::memcpy(out_cov, host + 3, 9 * sizeof(float));
  float ms = 0;
  if (cudaEventElapsedTime(&ms, m->ev[2], m->ev[3]) == cudaSuccess) m->last_ms[1] = ms;
  return B2S_OK;
}

b2s_status b2s_hector_map_copy(b2s_hector_map *m, float *log_odds, int32_t *update_index) {
  if (!m) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const size_t bytes = (size_t)m->sx * m->sy * 4;
  if (log_odds) B2S_CUDA_CHECK(cudaMemcpyAsync(log_odds, m->d_lo, bytes, cudaMemcpyDeviceToHost, m->stream));
  if (update_index) B2S_CUDA_CHECK(cudaMemcpyAsync(update_index, m->d_ui, bytes, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_hector_map_copy_ros(b2s_hector_map *m, int8_t *out) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int n = m->sx * m->sy;
  AsyncBuf<int8_t> d(m->stream);
  B2S_CUDA_CHECK(d.alloc((size_t)n));
  k_hector_ros<<<ceil_div(n, 256), 256, 0, m->stream>>>(m->d_lo, n, d);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, d, (size_t)n, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_hector_map_last_timing(b2s_hector_map *m, double out[2]) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  float ms = 0;
  if (cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]) == cudaSuccess) m->last_ms[0] = ms;
  out[0] = m->last_ms[0];
  out[1] = m->last_ms[1];
  return B2S_OK;
}

}  // extern "C"
