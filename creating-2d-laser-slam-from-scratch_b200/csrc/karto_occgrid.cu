// K2c — karto::OccupancyGrid::CreateFromScans on H100 (sm_90a).  Product code: CUDA only.
//
// Reference behaviour (paths relative to reference/lesson6/lib/open_karto/include/open_karto):
//   OccupancyGrid::{CreateFromScans, ComputeDimensions, AddScan, RayTrace, UpdateCell, Update}   Karto.h:5659-5673, 5804-5990
//   Grid<kt_int32u>::TraceLine                                                                Karto.h:4680-4745
//   LocalizedRangeScan::Update (bounding box, point readings)                                  Karto.h:5362-5428
//
// The whole map is rebuilt from ALL scans on every map publish (karto_slam.cc:511-512); the pass/hit counters are
// commutative uint32 sums, so every beam of every scan is independent: one warp per beam, lanes over the
// Bresenham steps.  TraceLine's error accumulator has the closed form
//     y(n) = y0 + ystep * floor((2*n*dy + dx) / (2*dx))        (n = step along the dominant axis)
// so each traversed cell is computed directly (no sequential dependency) and counted with a RED.ADD.
//
// HBM layout: pass[height][width_step] u32, hit[...] u32, cells[...] u8  (width_step = AlignValue(width, 8), the
// reference's own layout, so the buffers can be handed back verbatim).
// Algorithmic bytes (SURVEY.md §8(d)): A2 = 2 * 4 B * V, V = cell visits (end cell counted 3x: pass, pass, hit).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "karto_internal.cuh"
#include "nccl_dl.cuh"
#include "scan_kernels.cuh"

using namespace b2s;

struct b2s_occ_grid {
  Stream stream;
  b2s_occ_grid_info info;
  int device = 0;
  Buf<uint32_t> d_pass, d_hit;
  Buf<uint8_t> d_cells;
  double last_ms[2] = {0, 0};
};

namespace b2s {

// ---- the build: G grids, each CreateFromScans over its own scans, every stage one launch for all grids (the
// single-grid handle is a build of one grid).  Scans are numbered over all grids (grid 0's first); scan s reads row
// rows[s] of `ranges` (row s when rows is null) and belongs to grid scan_grid[s] (grid 0 when scan_grid is null).

struct OccGridDev {       // one grid of a build, as its kernels read it
  int w, h, step;
  int first, scans;       // the grid's first scan and its scan count
  double off_x, off_y, scale;
  long long counters;     // first counter of the grid in the pass / hit arena
  long long payload;      // first byte of its payload in the payload arena
};

// block-wide {min x, min y, max x, max y} of the threads' boxes into out[0..3]; one block of 256 threads
__device__ void bbox_reduce_block(double mnx, double mny, double mxx, double mxy, double *__restrict__ out) {
  __shared__ double sh[4][256];
  sh[0][threadIdx.x] = mnx; sh[1][threadIdx.x] = mny; sh[2][threadIdx.x] = mxx; sh[3][threadIdx.x] = mxy;
  __syncthreads();
  for (int d = blockDim.x / 2; d > 0; d >>= 1) {
    if (threadIdx.x < d) {
      sh[0][threadIdx.x] = fmin(sh[0][threadIdx.x], sh[0][threadIdx.x + d]);
      sh[1][threadIdx.x] = fmin(sh[1][threadIdx.x], sh[1][threadIdx.x + d]);
      sh[2][threadIdx.x] = fmax(sh[2][threadIdx.x], sh[2][threadIdx.x + d]);
      sh[3][threadIdx.x] = fmax(sh[3][threadIdx.x], sh[3][threadIdx.x + d]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[0] = sh[0][0]; out[1] = sh[1][0]; out[2] = sh[2][0]; out[3] = sh[3][0]; }
}

// per-scan bounding box over the sensor position and the FILTERED point readings
// (InRange(reading, minRange, rangeThreshold), Karto.h:5382,5400,5418-5424).  One block of 256 threads per scan.
template <class R>
__global__ void k_scan_bbox(const R *__restrict__ ranges, const int32_t *__restrict__ rows,
                            const double *__restrict__ sensor, const double *__restrict__ pts, b2s_laser l,
                            double *__restrict__ bbox) {
  const int s = blockIdx.x, n = l.n_readings;
  const R *r = ranges + (rows ? (size_t)rows[s] : (size_t)s) * n;
  const double *p = pts + (size_t)s * n * 2;
  const double big = 999999999999999999.99999;  // Karto.h:2765
  double mnx = big, mny = big, mxx = -big, mxy = -big;
  if (threadIdx.x == 0) {
    double x = sensor[3 * s], y = sensor[3 * s + 1];
    if (x < mnx) mnx = x;
    if (y < mny) mny = y;
    if (x > mxx) mxx = x;
    if (y > mxy) mxy = y;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double rr = (double)r[i];
    if (!(rr >= l.min_range && rr <= l.range_threshold)) continue;
    double x = p[(size_t)i * 2], y = p[(size_t)i * 2 + 1];
    if (x < mnx) mnx = x;
    if (y < mny) mny = y;
    if (x > mxx) mxx = x;
    if (y > mxy) mxy = y;
  }
  bbox_reduce_block(mnx, mny, mxx, mxy, bbox + 4 * s);
}

// union of each grid's scan boxes (OccupancyGrid::ComputeDimensions, Karto.h:5810-5814); one block of 256 threads per
// grid
__global__ void k_bbox_union(const double *__restrict__ bbox, const OccGridDev *__restrict__ grids,
                             double *__restrict__ out) {
  const int g = blockIdx.x, first = grids[g].first, scans = grids[g].scans;
  const double big = 999999999999999999.99999;
  double mnx = big, mny = big, mxx = -big, mxy = -big;
  for (int k = threadIdx.x; k < scans; k += blockDim.x) {
    const double *b = bbox + 4 * ((size_t)first + k);
    mnx = fmin(mnx, fmin(b[0], b[2]));  // Add(min); Add(max) (Karto.h:2824-2828)
    mny = fmin(mny, fmin(b[1], b[3]));
    mxx = fmax(mxx, fmax(b[0], b[2]));
    mxy = fmax(mxy, fmax(b[1], b[3]));
  }
  bbox_reduce_block(mnx, mny, mxx, mxy, out + 4 * g);
}

// OccupancyGrid::AddScan + RayTrace + Grid::TraceLine (Karto.h:5852-5945, 4680-4745) for ONE beam, by one warp: the
// lanes split the Bresenham steps.  Returns the cell visits this lane counted.
__device__ __forceinline__ unsigned long long trace_beam(double rr, double sx, double sy, double px, double py,
                                                         const b2s_laser &l, int w, int h, int step, double off_x,
                                                         double off_y, double scale, int lane, uint32_t *__restrict__ pass,
                                                         uint32_t *__restrict__ hit) {
  if (rr <= l.min_range || rr >= l.max_range || isnan(rr)) return 0;  // Karto.h:5873-5878
  unsigned long long visits = 0;
  const bool end_valid = rr < (l.range_threshold - KT_TOLERANCE);     // Karto.h:5871
  if (rr >= l.range_threshold) {  // Karto.h:5879-5887: clip to the range threshold, no hit
    const double ratio = l.range_threshold / rr;
    const double dx = px - sx, dy = py - sy;
    px = __dadd_rn(sx, __dmul_rn(ratio, dx));
    py = __dadd_rn(sy, __dmul_rn(ratio, dy));
  }
  int x0 = world_to_grid_1(sx, off_x, scale), y0 = world_to_grid_1(sy, off_y, scale);
  int x1 = world_to_grid_1(px, off_x, scale), y1 = world_to_grid_1(py, off_y, scale);
  // the end cell (Karto.h:5924-5942), counted before the walk so that its coordinates hold no register during it (the
  // counters are sums: the order does not matter)
  if (lane == 0 && end_valid && x1 >= 0 && x1 < w && y1 >= 0 && y1 < h) {
    atomicAdd(pass + x1 + (size_t)y1 * step, 1u);
    atomicAdd(hit + x1 + (size_t)y1 * step, 1u);
    visits += 2;
  }
  // TraceLine canonicalisation (Karto.h:4682-4692)
  const bool steep = abs(y1 - y0) > abs(x1 - x0);
  if (steep) { int t = x0; x0 = y0; y0 = t; t = x1; x1 = y1; y1 = t; }
  if (x0 > x1) { int t = x0; x0 = x1; x1 = t; t = y0; y0 = y1; y1 = t; }
  const long long dx = (long long)x1 - x0, dy = llabs((long long)y1 - y0);
  const int ystep = (y0 < y1) ? 1 : -1;
  for (long long k = lane; k <= dx; k += 32) {
    // y before the update of step k: increments so far = floor((2*k*dy + dx) / (2*dx))  (0 when dx == 0)
    const long long inc = dx > 0 ? (2 * k * dy + dx) / (2 * dx) : 0;
    const int x = x0 + (int)k, y = y0 + ystep * (int)inc;
    const int cx = steep ? y : x, cy = steep ? x : y;
    if (cx >= 0 && cx < w && cy >= 0 && cy < h) {
      atomicAdd(pass + cx + (size_t)cy * step, 1u);
      visits++;
    }
  }
  return visits;
}

// the warp's visit counts added to *to by lane 0: one atomic per warp
__device__ __forceinline__ void add_warp_visits(unsigned long long v, int lane, unsigned long long *__restrict__ to) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  if (lane == 0 && v) atomicAdd(to, v);
}

// every beam of every scan of every grid, one warp per beam.  A lane sums its cell visits in a register; the warp adds
// them to visits[g] when its next beam belongs to another grid, and once at the end, so a build of one grid costs one
// atomic per warp.  48 registers, no spills (-Xptxas -v): 5 CTAs per SM.
template <class R>
__global__ void __launch_bounds__(256, 5)
    k_raytrace(const R *__restrict__ ranges, const int32_t *__restrict__ rows, const int32_t *__restrict__ scan_grid,
               const double *__restrict__ sensor, const double *__restrict__ pts, b2s_laser l, long long n_beams,
               const OccGridDev *__restrict__ grids, uint32_t *__restrict__ pass, uint32_t *__restrict__ hit,
               unsigned long long *__restrict__ visits) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n = l.n_readings;
  int g = -1;  // warp-uniform
  OccGridDev G{};
  unsigned long long my_visits = 0;
  for (long long beam = warp0; beam < n_beams; beam += nwarps) {
    const int s = (int)(beam / n), i = (int)(beam - (long long)s * n);
    const int gs = scan_grid ? scan_grid[s] : 0;
    if (gs != g) {
      if (g >= 0) add_warp_visits(my_visits, lane, visits + g);
      my_visits = 0;
      g = gs;
      G = grids[g];
    }
    if (G.w <= 0 || G.h <= 0) continue;
    const size_t row = rows ? (size_t)rows[s] : (size_t)s;
    my_visits += trace_beam((double)ranges[row * n + i], sensor[3 * s], sensor[3 * s + 1], pts[beam * 2],
                            pts[beam * 2 + 1], l, G.w, G.h, G.step, G.off_x, G.off_y, G.scale, lane, pass + G.counters,
                            hit + G.counters);
  }
  if (g >= 0) add_warp_visits(my_visits, lane, visits + g);
}

// ---- thresholds and ROS payloads

// OccupancyGrid::UpdateCell (Karto.h:5970-5990): MinPassThrough = 2, OccupancyThreshold = 0.1
__device__ __forceinline__ uint8_t occ_cell_value(uint32_t p, uint32_t h) {
  uint8_t v = 0;
  if (p > 2u) {
    const double ratio = (double)h / (double)p;
    v = ratio > 0.1 ? (uint8_t)GRID_OCCUPIED : (uint8_t)GRID_FREE;
  }
  return v;
}

// SlamKarto::updateMap payload (karto_slam.cc:546-569): unknown -> -1, occupied -> 100, free -> 0
__device__ __forceinline__ int8_t occ_ros_value(uint8_t v) { return v == 0 ? -1 : (v == GRID_OCCUPIED ? 100 : 0); }

// OccupancyGrid::Update (Karto.h:5953-5968)
__global__ void k_occ_threshold(const uint32_t *__restrict__ pass, const uint32_t *__restrict__ hit, int n,
                                uint8_t *__restrict__ cells) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  cells[i] = occ_cell_value(pass[i], hit[i]);
}

// row-major w x h payload
__global__ void k_occ_ros(const uint8_t *__restrict__ cells, int w, int h, int step, int8_t *__restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const int x = i % w, y = i / w;
  out[i] = occ_ros_value(cells[x + (size_t)y * step]);
}

// thresholds and ROS payload of every grid: grids blockIdx.y, + gridDim.y, ... (grid_rows(n_grids) rows), x-blocks
// stride over each one's w x h cells
__global__ void k_occ_ros_grids(const uint32_t *__restrict__ pass, const uint32_t *__restrict__ hit,
                                const OccGridDev *__restrict__ grids, int n_grids, int8_t *__restrict__ out) {
  for (int g = blockIdx.y; g < n_grids; g += gridDim.y) {
    const OccGridDev G = grids[g];
    const long long cells = (long long)G.w * G.h;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (long long)gridDim.x * blockDim.x) {
      const int x = (int)(i % G.w), y = (int)(i / G.w);
      const size_t c = (size_t)G.counters + x + (size_t)y * G.step;
      out[G.payload + i] = occ_ros_value(occ_cell_value(pass[c], hit[c]));
    }
  }
}

}  // namespace b2s

// OccupancyGrid::ComputeDimensions (Karto.h:5816-5821) from the scans' box {min x, min y, max x, max y}
static b2s_status occ_dims(const double bb[4], double resolution, b2s_occ_grid_info &I) {
  const double scale = 1.0 / resolution;
  I.width = cast_i32(kround((bb[2] - bb[0]) * scale));
  I.height = cast_i32(kround((bb[3] - bb[1]) * scale));
  // the counters hold width_step * height cells (rows padded to 8), indexed and sized in int32
  if (I.width < 0 || I.height < 0 || I.width > INT32_MAX - 7 || ((long long)I.width + 7) / 8 * 8 * I.height > INT32_MAX)
    B2S_FAIL(B2S_ERR_TOO_LARGE, "occupancy grid dimensions out of range");
  I.width_step = (I.width + 7) & ~7;
  I.data_size = I.width_step * I.height;
  I.offset[0] = bb[0];
  I.offset[1] = bb[1];
  I.resolution = resolution;
  I.cell_visits = 0;
  return B2S_OK;
}

extern "C" void b2s_occ_grid_destroy(b2s_occ_grid *g);
extern "C" {

// given_bbox == nullptr: CreateFromScans (the box is the union over these scans).  given_bbox != nullptr: the scans
// are one SHARD of a scan list whose global box the caller has reduced over all shards (SURVEY.md §8(e)(iii)); the
// counters then hold this shard's contribution only.  bbox_out != nullptr: compute the shard's box and stop.
static b2s_status occ_create_impl(const b2s_laser *laser, int n_scans, const double *ranges, const double *poses,
                                  double resolution, const double *given_bbox, double *bbox_out, int device,
                                  void *cuda_stream, b2s_occ_grid **out) {
  B2S_NVTX("K2c OccupancyGrid::CreateFromScans");
  if (!laser || n_scans < 0 || (n_scans > 0 && (!ranges || !poses)) || (!out && !bbox_out))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid: null/negative argument");
  if (out) *out = nullptr;
  if (n_scans == 0 && !given_bbox && !bbox_out) return B2S_OK;  // CreateFromScans returns NULL for an empty scan list (Karto.h:5661-5664)
  if (bbox_out && n_scans == 0) {  // BoundingBox2 of nothing (Karto.h:2765-2770)
    const double big = 999999999999999999.99999;
    bbox_out[0] = big; bbox_out[1] = big; bbox_out[2] = -big; bbox_out[3] = -big;
    return B2S_OK;
  }
  if (double_equal(resolution, 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "Resolution cannot be 0");  // Karto.h:5627-5630
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<b2s_occ_grid, decltype(&b2s_occ_grid_destroy)> g(new (std::nothrow) b2s_occ_grid(), b2s_occ_grid_destroy);
  if (!g) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  g->device = device;
  B2S_CUDA_CHECK(g->stream.init(cuda_stream));
  cudaStream_t st = g->stream;
  const size_t n = (size_t)std::max(laser->n_readings, 0), M = (size_t)n_scans;
  Event ev[3];
  for (auto &e : ev) B2S_CUDA_CHECK(e.create());
  AsyncBuf<double> d_ranges(st), d_poses(st), d_sensor(st), d_pts(st), d_bbox(st);
  AsyncBuf<unsigned long long> d_visits(st);
  AsyncBuf<OccGridDev> d_grid(st);
  B2S_CUDA_CHECK(d_ranges.alloc(std::max<size_t>(M * n, 1)));
  B2S_CUDA_CHECK(d_poses.alloc(std::max<size_t>(M * 3, 1)));
  B2S_CUDA_CHECK(d_sensor.alloc(std::max<size_t>(M * 3, 1)));
  B2S_CUDA_CHECK(d_pts.alloc(std::max<size_t>(M * n * 2, 1)));
  B2S_CUDA_CHECK(d_bbox.alloc((M + 1) * 4));
  B2S_CUDA_CHECK(d_visits.alloc(1));
  B2S_CUDA_CHECK(d_grid.alloc(1));
  if (n && M) B2S_CUDA_CHECK(cudaMemcpyAsync(d_ranges, ranges, sizeof(double) * M * n, cudaMemcpyHostToDevice, st));
  if (M) B2S_CUDA_CHECK(cudaMemcpyAsync(d_poses, poses, sizeof(double) * M * 3, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemsetAsync(d_visits, 0, sizeof(unsigned long long), st));
  // a build of one grid: scan s is row s of d_ranges, counters and payload start at 0
  OccGridDev D{};
  D.scans = n_scans;
  double bb[4];
  if (M) k_scan_points<<<(unsigned)M, 256, 0, st>>>(d_ranges, d_poses, *laser, d_sensor, d_pts, nullptr, nullptr);
  if (given_bbox) {
    for (int i = 0; i < 4; i++) bb[i] = given_bbox[i];
  } else {
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_grid, &D, sizeof(D), cudaMemcpyHostToDevice, st));
    k_scan_bbox<<<(unsigned)M, 256, 0, st>>>((const double *)d_ranges, nullptr, d_sensor, d_pts, *laser, d_bbox);
    k_bbox_union<<<1, 256, 0, st>>>(d_bbox, d_grid, d_bbox + 4 * M);
    B2S_CUDA_CHECK(cudaGetLastError());
    B2S_CUDA_CHECK(cudaMemcpyAsync(bb, d_bbox + 4 * M, sizeof(bb), cudaMemcpyDeviceToHost, st));
    B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  if (bbox_out) {
    for (int i = 0; i < 4; i++) bbox_out[i] = bb[i];
    return B2S_OK;
  }
  b2s_occ_grid_info &I = g->info;
  if (b2s_status s = occ_dims(bb, resolution, I)) return s;
  D.w = I.width; D.h = I.height; D.step = I.width_step;
  D.off_x = I.offset[0]; D.off_y = I.offset[1]; D.scale = 1.0 / resolution;
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_grid, &D, sizeof(D), cudaMemcpyHostToDevice, st));
  const size_t cells = (size_t)std::max(I.data_size, 1);
  B2S_CUDA_CHECK(g->d_pass.reserve(cells));
  B2S_CUDA_CHECK(g->d_hit.reserve(cells));
  B2S_CUDA_CHECK(g->d_cells.reserve(cells));
  B2S_CUDA_CHECK(cudaMemsetAsync(g->d_pass, 0, sizeof(uint32_t) * cells, st));
  B2S_CUDA_CHECK(cudaMemsetAsync(g->d_hit, 0, sizeof(uint32_t) * cells, st));
  B2S_CUDA_CHECK(cudaEventRecord(ev[0], st));
  if (n && M && I.data_size > 0) {
    const long long n_beams = (long long)M * (long long)n;
    const int sms = sm_count(device);
    // Global RED.ADD.  (A shared-memory privatised variant — row bands of the map as per-CTA uint32 tiles, lines clipped
    // to a band in closed form — was built and measured slower (not re-measured on the H100): shared-memory atomics
    // retire no faster than the L2 atomic units, and one 200 KB tile per SM leaves few warps to hide their latency.)
    const int blocks = (int)std::min<long long>((n_beams + 7) / 8, (long long)sms * 16);
    k_raytrace<<<blocks, 256, 0, st>>>((const double *)d_ranges, nullptr, nullptr, d_sensor, d_pts, *laser, n_beams,
                                       d_grid, g->d_pass, g->d_hit, d_visits);
  }
  B2S_CUDA_CHECK(cudaEventRecord(ev[1], st));
  if (I.data_size > 0) k_occ_threshold<<<ceil_div(I.data_size, 256), 256, 0, st>>>(g->d_pass, g->d_hit, I.data_size, g->d_cells);
  B2S_CUDA_CHECK(cudaEventRecord(ev[2], st));
  B2S_CUDA_CHECK(cudaGetLastError());
  unsigned long long visits = 0;
  B2S_CUDA_CHECK(cudaMemcpyAsync(&visits, d_visits, sizeof(visits), cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  I.cell_visits = visits;
  float ms = 0;
  if (cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) g->last_ms[0] = ms;
  if (cudaEventElapsedTime(&ms, ev[1], ev[2]) == cudaSuccess) g->last_ms[1] = ms;
  *out = g.release();
  return B2S_OK;
}

b2s_status b2s_occ_grid_create_from_scans(const b2s_laser *laser, int n_scans, const double *ranges,
                                          const double *poses, double resolution, int device, void *cuda_stream,
                                          b2s_occ_grid **out) {
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_create_from_scans: null argument");
  return occ_create_impl(laser, n_scans, ranges, poses, resolution, nullptr, nullptr, device, cuda_stream, out);
}

b2s_status b2s_occ_grid_scans_bbox(const b2s_laser *laser, int n_scans, const double *ranges, const double *poses,
                                   int device, void *cuda_stream, double bbox[4]) {
  if (!bbox) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_scans_bbox: null argument");
  return occ_create_impl(laser, n_scans, ranges, poses, 1.0, nullptr, bbox, device, cuda_stream, nullptr);
}

b2s_status b2s_occ_grid_create_shard(const b2s_laser *laser, int n_scans, const double *ranges, const double *poses,
                                     double resolution, const double bbox[4], int device, void *cuda_stream,
                                     b2s_occ_grid **out) {
  if (!out || !bbox) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_create_shard: null argument");
  return occ_create_impl(laser, n_scans, ranges, poses, resolution, bbox, nullptr, device, cuda_stream, out);
}

b2s_status b2s_occ_grid_device_counters(b2s_occ_grid *g, uint32_t **d_pass, uint32_t **d_hit) {
  if (!g || !d_pass || !d_hit) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));  // the caller's collective runs on its own stream
  *d_pass = g->d_pass;
  *d_hit = g->d_hit;
  return B2S_OK;
}

/* step 3 of the sharded build with the collective inside the library: pass / hit counters summed over the ranks in place
 * on the device (two ncclAllReduce(SUM, uint32) on the grid's stream through the caller's communicator) */
b2s_status b2s_occ_grid_allreduce_counters(b2s_occ_grid *g, void *nccl_comm) {
  if (!g || !nccl_comm) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  const NcclApi &nc = nccl_api();
  if (!nc.ok) B2S_FAIL(B2S_ERR_BAD_STATE, "libnccl.so.2 could not be loaded (dlopen)");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const size_t cells = (size_t)std::max(g->info.data_size, 0);
  if (cells == 0) return B2S_OK;
  for (uint32_t *buf : {g->d_pass.p, g->d_hit.p}) {
    const int rc = nc.all_reduce(buf, buf, cells, NCCL_UINT32, NCCL_SUM, nccl_comm, g->stream);
    if (rc != 0) B2S_FAIL(B2S_ERR_CUDA, std::string("ncclAllReduce(counters) failed: ") + (nc.error_string ? nc.error_string(rc) : "NCCL error"));
  }
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

b2s_status b2s_occ_grid_set_counters(b2s_occ_grid *g, const uint32_t *pass, const uint32_t *hit) {
  if (!g || !pass || !hit) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const size_t n = (size_t)g->info.data_size;
  if (n) {
    B2S_CUDA_CHECK(cudaMemcpyAsync(g->d_pass, pass, n * sizeof(uint32_t), cudaMemcpyHostToDevice, g->stream));
    B2S_CUDA_CHECK(cudaMemcpyAsync(g->d_hit, hit, n * sizeof(uint32_t), cudaMemcpyHostToDevice, g->stream));
    B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  }
  return B2S_OK;
}

b2s_status b2s_occ_grid_update(b2s_occ_grid *g) {  // OccupancyGrid::Update (Karto.h:5953-5968)
  if (!g) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const int n = g->info.data_size;
  if (n > 0) k_occ_threshold<<<ceil_div(n, 256), 256, 0, g->stream>>>(g->d_pass, g->d_hit, n, g->d_cells);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

b2s_status b2s_occ_grid_info_get(const b2s_occ_grid *g, b2s_occ_grid_info *out) {
  if (!g || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  *out = g->info;
  return B2S_OK;
}

b2s_status b2s_occ_grid_copy(b2s_occ_grid *g, uint8_t *cells, uint32_t *pass, uint32_t *hit) {
  if (!g) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const size_t n = (size_t)g->info.data_size;
  if (cells && n) B2S_CUDA_CHECK(cudaMemcpyAsync(cells, g->d_cells, n, cudaMemcpyDeviceToHost, g->stream));
  if (pass && n) B2S_CUDA_CHECK(cudaMemcpyAsync(pass, g->d_pass, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, g->stream));
  if (hit && n) B2S_CUDA_CHECK(cudaMemcpyAsync(hit, g->d_hit, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, g->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

b2s_status b2s_occ_grid_copy_ros(b2s_occ_grid *g, int8_t *out) {
  if (!g || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const int w = g->info.width, h = g->info.height;
  if (w * h == 0) return B2S_OK;
  AsyncBuf<int8_t> d(g->stream);
  B2S_CUDA_CHECK(d.alloc((size_t)w * h));
  k_occ_ros<<<ceil_div((long long)w * h, 256), 256, 0, g->stream>>>(g->d_cells, w, h, g->info.width_step, d);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, d, (size_t)w * h, cudaMemcpyDeviceToHost, g->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

b2s_status b2s_occ_grid_last_timing(b2s_occ_grid *g, double out[2]) {
  if (!g || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  out[0] = g->last_ms[0];
  out[1] = g->last_ms[1];
  return B2S_OK;
}

void b2s_occ_grid_destroy(b2s_occ_grid *g) {
  if (!g) return;
  cudaSetDevice(g->device);
  cudaStreamSynchronize(g->stream);
  delete g;
}

}  // extern "C"

// ---- batched builds: CreateFromScans for many grids at once over a device-resident float32 pool of readings
namespace b2s {

struct OccBatch {
  Stream stream;  // first: destroyed last
  int device = 0;
  b2s_laser laser{};
  Buf<float> d_pool;                 // [pool_rows][n_readings] readings, each uploaded once
  size_t pool_rows = 0;
  HostBuf<float> h_stage;            // page-locked staging of appended rows
  Buf<int32_t> d_rows, d_scan_grid;
  Buf<double> d_poses, d_sensor, d_pts, d_bbox, d_union;
  Buf<OccGridDev> d_grids;
  Buf<uint32_t> d_pass, d_hit;       // one arena of counters for every grid of a build
  Buf<unsigned long long> d_visits;
  Buf<int8_t> d_payload;
  HostBuf<int32_t> h_i32;            // rows, scan_grid of a build
  HostBuf<double> h_f64;             // poses of a build; the unions read back
  HostBuf<OccGridDev> h_grids;
  HostBuf<unsigned long long> h_visits;
  HostBuf<int8_t> h_payload;         // every payload of the last build
  std::vector<OccGridDev> grids;
  double bytes_d2h = 0;              // read back over the handle's life
};

b2s_status occ_batch_create(const b2s_laser &laser, int device, OccBatch **out) {
  *out = nullptr;
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<OccBatch> b(new (std::nothrow) OccBatch());
  if (!b) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  b->device = device;
  b->laser = laser;
  B2S_CUDA_CHECK(b->stream.init(nullptr));
  *out = b.release();
  return B2S_OK;
}

void occ_batch_destroy(OccBatch *b) {
  if (!b) return;
  cudaSetDevice(b->device);
  cudaStreamSynchronize(b->stream);
  delete b;
}

double occ_batch_bytes_d2h(const OccBatch *b) { return b ? b->bytes_d2h : 0.0; }

// rows [count][n_readings] (host) appended to the pool in one copy; *first = the first new row
b2s_status occ_batch_append(OccBatch *b, int count, const float *rows, int32_t *first) {
  const size_t n = (size_t)std::max(b->laser.n_readings, 1);
  *first = (int32_t)b->pool_rows;
  if (count <= 0) return B2S_OK;
  if (b->pool_rows + (size_t)count > (size_t)INT32_MAX) B2S_FAIL(B2S_ERR_TOO_LARGE, "occupancy grid pool: too many scans");
  B2S_CUDA_CHECK(cudaSetDevice(b->device));
  cudaStream_t st = b->stream;
  if ((b->pool_rows + count) * n > b->d_pool.cap) {  // full: twice the rows (256 at first)
    Buf<float> fresh;
    B2S_CUDA_CHECK(fresh.reserve(std::max<size_t>(std::max<size_t>(256, 2 * b->pool_rows), b->pool_rows + count) * n));
    if (b->pool_rows)
      B2S_CUDA_CHECK(cudaMemcpyAsync(fresh, b->d_pool, sizeof(float) * b->pool_rows * n, cudaMemcpyDeviceToDevice, st));
    B2S_CUDA_CHECK(cudaStreamSynchronize(st));
    b->d_pool = std::move(fresh);
  }
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));  // the staging buffer is free again
  B2S_CUDA_CHECK(b->h_stage.reserve((size_t)count * n));
  std::memcpy(b->h_stage, rows, sizeof(float) * (size_t)count * (size_t)b->laser.n_readings);
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->d_pool + b->pool_rows * n, b->h_stage, sizeof(float) * count * n,
                                 cudaMemcpyHostToDevice, st));
  b->pool_rows += (size_t)count;
  return B2S_OK;
}

// G grids, grid g = CreateFromScans over n_scans[g] scans: pool rows rows[], robot poses poses[][3] (grid 0's scans
// first) at resolution[g].  have[g] = 0 when the grid has no scans (CreateFromScans returns NULL), else info[g] and
// payload[g] (valid until the next build) are its map.
b2s_status occ_batch_build(OccBatch *b, int G, const int32_t *n_scans, const int32_t *rows, const double *poses,
                           const double *resolution, b2s_occ_grid_info *info, int32_t *have, const int8_t **payload) {
  B2S_NVTX("K2c OccupancyGrid::CreateFromScans, batched");
  const b2s_laser &l = b->laser;
  const size_t n = (size_t)std::max(l.n_readings, 0);
  size_t M = 0;
  for (int g = 0; g < G; g++) {
    have[g] = n_scans[g] > 0;
    payload[g] = nullptr;
    M += (size_t)std::max(n_scans[g], 0);
    if (n_scans[g] > 0 && double_equal(resolution[g], 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "Resolution cannot be 0");
  }
  if (M == 0) return B2S_OK;
  B2S_CUDA_CHECK(cudaSetDevice(b->device));
  cudaStream_t st = b->stream;
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));  // the page-locked buffers of the previous build are free
  // the build's scans: pool rows, poses, and per grid its first scan and count (grids without scans are left out)
  std::vector<int> live;
  for (int g = 0; g < G; g++)
    if (n_scans[g] > 0) live.push_back(g);
  const int L = (int)live.size();
  B2S_CUDA_CHECK(b->h_i32.reserve(2 * M));
  B2S_CUDA_CHECK(b->h_f64.reserve(std::max<size_t>(3 * M, 4 * (size_t)L)));
  B2S_CUDA_CHECK(b->d_grids.reserve((size_t)L));
  B2S_CUDA_CHECK(b->h_grids.reserve((size_t)L));
  int32_t *h_rows = b->h_i32, *h_grid = h_rows + M;
  b->grids.assign((size_t)L, OccGridDev{});
  {
    size_t s = 0;
    for (int j = 0; j < L; j++) {
      const int g = live[(size_t)j];
      b->grids[(size_t)j].first = (int)s;
      b->grids[(size_t)j].scans = n_scans[g];
      for (int k = 0; k < n_scans[g]; k++) h_grid[s + k] = j;
      s += (size_t)n_scans[g];
    }
  }
  auto upload_grids = [&] {
    std::memcpy(b->h_grids, b->grids.data(), sizeof(OccGridDev) * L);
    return cudaMemcpyAsync(b->d_grids, b->h_grids, sizeof(OccGridDev) * L, cudaMemcpyHostToDevice, st);
  };
  {
    size_t s = 0;
    for (int g = 0, src = 0; g < G; g++) {
      const size_t c = (size_t)std::max(n_scans[g], 0);
      if (c) {
        std::memcpy(h_rows + s, rows + src, sizeof(int32_t) * c);
        std::memcpy((double *)b->h_f64 + 3 * s, poses + 3 * (size_t)src, sizeof(double) * 3 * c);
        s += c;
      }
      src += (int)c;
    }
  }
  for (size_t s = 0; s < M; s++)
    if (h_rows[s] < 0 || (size_t)h_rows[s] >= b->pool_rows) B2S_FAIL(B2S_ERR_OUT_OF_RANGE, "occupancy grid pool row out of range");
  B2S_CUDA_CHECK(b->d_rows.reserve(M));
  B2S_CUDA_CHECK(b->d_scan_grid.reserve(M));
  B2S_CUDA_CHECK(b->d_poses.reserve(3 * M));
  B2S_CUDA_CHECK(b->d_sensor.reserve(3 * M));
  B2S_CUDA_CHECK(b->d_pts.reserve(M * std::max<size_t>(n, 1) * 2));
  B2S_CUDA_CHECK(b->d_bbox.reserve(4 * M));
  B2S_CUDA_CHECK(b->d_union.reserve(4 * (size_t)L));
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->d_rows, h_rows, sizeof(int32_t) * M, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->d_scan_grid, h_grid, sizeof(int32_t) * M, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(upload_grids());
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->d_poses, b->h_f64, sizeof(double) * 3 * M, cudaMemcpyHostToDevice, st));
  // points, per-scan boxes, per-grid unions, then the unions back to size the grids on the host
  k_scan_points<<<(unsigned)M, 256, 0, st>>>((const float *)b->d_pool, (const double *)b->d_poses, l, b->d_sensor.p,
                                             b->d_pts.p, nullptr, (const int32_t *)b->d_rows);
  k_scan_bbox<<<(unsigned)M, 256, 0, st>>>((const float *)b->d_pool, b->d_rows, b->d_sensor, b->d_pts, l, b->d_bbox);
  k_bbox_union<<<(unsigned)L, 256, 0, st>>>(b->d_bbox, b->d_grids, b->d_union);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->h_f64, b->d_union, sizeof(double) * 4 * L, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  b->bytes_d2h += sizeof(double) * 4.0 * L;
  long long counters = 0, bytes = 0;
  for (int j = 0; j < L; j++) {
    const int g = live[(size_t)j];
    if (b2s_status s = occ_dims((const double *)b->h_f64 + 4 * j, resolution[g], info[g])) return s;
    OccGridDev &D = b->grids[(size_t)j];
    D.w = info[g].width; D.h = info[g].height; D.step = info[g].width_step;
    D.off_x = info[g].offset[0]; D.off_y = info[g].offset[1]; D.scale = 1.0 / resolution[g];
    D.counters = counters;
    D.payload = bytes;
    counters += info[g].data_size;
    bytes += (long long)D.w * D.h;
  }
  B2S_CUDA_CHECK(b->d_pass.reserve((size_t)counters));
  B2S_CUDA_CHECK(b->d_hit.reserve((size_t)counters));
  B2S_CUDA_CHECK(b->d_visits.reserve((size_t)L));
  B2S_CUDA_CHECK(b->d_payload.reserve((size_t)bytes));
  B2S_CUDA_CHECK(b->h_payload.reserve((size_t)bytes));
  B2S_CUDA_CHECK(b->h_visits.reserve((size_t)L));
  B2S_CUDA_CHECK(upload_grids());
  if (counters) {
    B2S_CUDA_CHECK(cudaMemsetAsync(b->d_pass, 0, sizeof(uint32_t) * counters, st));
    B2S_CUDA_CHECK(cudaMemsetAsync(b->d_hit, 0, sizeof(uint32_t) * counters, st));
  }
  B2S_CUDA_CHECK(cudaMemsetAsync(b->d_visits, 0, sizeof(unsigned long long) * L, st));
  const long long n_beams = (long long)M * (long long)n;
  if (n_beams && counters) {
    const int blocks = (int)std::min<long long>((n_beams + 7) / 8, (long long)sm_count(b->device) * 16);
    k_raytrace<<<blocks, 256, 0, st>>>((const float *)b->d_pool, b->d_rows, b->d_scan_grid, b->d_sensor, b->d_pts, l,
                                       n_beams, b->d_grids, b->d_pass, b->d_hit, b->d_visits);
  }
  if (bytes) {
    long long most = 0;
    for (const OccGridDev &D : b->grids) most = std::max(most, (long long)D.w * D.h);
    const unsigned xb = (unsigned)std::min<long long>(ceil_div(most, 256), 1024);
    k_occ_ros_grids<<<dim3(xb, grid_rows(L)), 256, 0, st>>>(b->d_pass, b->d_hit, b->d_grids, L, b->d_payload);
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  if (bytes) B2S_CUDA_CHECK(cudaMemcpyAsync(b->h_payload, b->d_payload, (size_t)bytes, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(b->h_visits, b->d_visits, sizeof(unsigned long long) * L, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  b->bytes_d2h += (double)bytes + sizeof(unsigned long long) * (double)L;
  for (int j = 0; j < L; j++) {
    const int g = live[(size_t)j];
    info[g].cell_visits = b->h_visits[j];
    payload[g] = (const int8_t *)b->h_payload + b->grids[(size_t)j].payload;
  }
  return B2S_OK;
}

}  // namespace b2s

extern "C" b2s_status b2s_occ_grid_create_from_scans_batch(const b2s_laser *laser, int n_grids, const int32_t *n_scans,
                                                           const float *ranges, const double *poses,
                                                           const double *resolution, int device,
                                                           b2s_occ_grid_batch_fn on_grid, void *user) {
  if (!laser || n_grids < 0 || (n_grids > 0 && (!n_scans || !resolution)))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_create_from_scans_batch: null argument or negative count");
  size_t M = 0;
  for (int g = 0; g < n_grids; g++) {
    if (n_scans[g] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_create_from_scans_batch: negative scan count");
    M += (size_t)n_scans[g];
  }
  if (M > (size_t)INT32_MAX) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_occ_grid_create_from_scans_batch: too many scans");
  if (M > 0 && (!ranges || !poses)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_occ_grid_create_from_scans_batch: null argument");
  if (M == 0) return B2S_OK;
  OccBatch *raw = nullptr;
  if (b2s_status st = occ_batch_create(*laser, device, &raw)) return st;
  std::unique_ptr<OccBatch, decltype(&occ_batch_destroy)> b(raw, occ_batch_destroy);
  int32_t first = 0;
  if (b2s_status st = occ_batch_append(b.get(), (int)M, ranges, &first)) return st;
  std::vector<int32_t> rows(M), have((size_t)n_grids);
  for (size_t s = 0; s < M; s++) rows[s] = first + (int32_t)s;
  std::vector<b2s_occ_grid_info> info((size_t)n_grids);
  std::vector<const int8_t *> payload((size_t)n_grids);
  if (b2s_status st = occ_batch_build(b.get(), n_grids, n_scans, rows.data(), poses, resolution, info.data(),
                                      have.data(), payload.data()))
    return st;
  if (on_grid)
    for (int g = 0; g < n_grids; g++)
      if (have[(size_t)g]) on_grid(user, g, &info[(size_t)g], payload[(size_t)g]);
  return B2S_OK;
}
