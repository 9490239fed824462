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

// per-scan bounding box over the sensor position and the FILTERED point readings
// (InRange(reading, minRange, rangeThreshold), Karto.h:5382,5400,5418-5424).  One block per scan.
__global__ void k_scan_bbox(const double *__restrict__ ranges, const double *__restrict__ sensor,
                            const double *__restrict__ pts, b2s_laser l, double *__restrict__ bbox) {
  const int s = blockIdx.x, n = l.n_readings;
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
    double r = ranges[(size_t)s * n + i];
    if (!(r >= l.min_range && r <= l.range_threshold)) continue;
    double x = pts[((size_t)s * n + i) * 2], y = pts[((size_t)s * n + i) * 2 + 1];
    if (x < mnx) mnx = x;
    if (y < mny) mny = y;
    if (x > mxx) mxx = x;
    if (y > mxy) mxy = y;
  }
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
  if (threadIdx.x == 0) {
    bbox[4 * s] = sh[0][0]; bbox[4 * s + 1] = sh[1][0]; bbox[4 * s + 2] = sh[2][0]; bbox[4 * s + 3] = sh[3][0];
  }
}

// union of the per-scan boxes (OccupancyGrid::ComputeDimensions, Karto.h:5810-5814); single block
__global__ void k_bbox_union(const double *__restrict__ bbox, int n_scans, double *__restrict__ out) {
  const double big = 999999999999999999.99999;
  double mnx = big, mny = big, mxx = -big, mxy = -big;
  for (int s = threadIdx.x; s < n_scans; s += blockDim.x) {
    mnx = fmin(mnx, fmin(bbox[4 * s], bbox[4 * s + 2]));  // Add(min); Add(max) (Karto.h:2824-2828)
    mny = fmin(mny, fmin(bbox[4 * s + 1], bbox[4 * s + 3]));
    mxx = fmax(mxx, fmax(bbox[4 * s], bbox[4 * s + 2]));
    mxy = fmax(mxy, fmax(bbox[4 * s + 1], bbox[4 * s + 3]));
  }
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

// OccupancyGrid::AddScan + RayTrace + Grid::TraceLine (Karto.h:5852-5945, 4680-4745).  One warp per beam.
__global__ void __launch_bounds__(256)
    k_raytrace(const double *__restrict__ ranges, const double *__restrict__ sensor, const double *__restrict__ pts,
               b2s_laser l, long long n_beams, int w, int h, int step, double off_x, double off_y, double scale,
               uint32_t *__restrict__ pass, uint32_t *__restrict__ hit, unsigned long long *__restrict__ visits) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int n = l.n_readings;
  unsigned long long my_visits = 0;
  for (long long beam = warp0; beam < n_beams; beam += nwarps) {
    const int s = (int)(beam / n);
    const double rr = ranges[beam];
    if (rr <= l.min_range || rr >= l.max_range || isnan(rr)) continue;  // Karto.h:5873-5878
    const bool end_valid = rr < (l.range_threshold - KT_TOLERANCE);     // Karto.h:5871
    const double sx = sensor[3 * s], sy = sensor[3 * s + 1];
    double px = pts[beam * 2], py = pts[beam * 2 + 1];
    if (rr >= l.range_threshold) {  // Karto.h:5879-5887: clip to the range threshold, no hit
      const double ratio = l.range_threshold / rr;
      const double dx = px - sx, dy = py - sy;
      px = __dadd_rn(sx, __dmul_rn(ratio, dx));
      py = __dadd_rn(sy, __dmul_rn(ratio, dy));
    }
    int x0 = world_to_grid_1(sx, off_x, scale), y0 = world_to_grid_1(sy, off_y, scale);
    int x1 = world_to_grid_1(px, off_x, scale), y1 = world_to_grid_1(py, off_y, scale);
    const int tx = x1, ty = y1;
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
        my_visits++;
      }
    }
    if (lane == 0 && end_valid && tx >= 0 && tx < w && ty >= 0 && ty < h) {  // Karto.h:5924-5942
      atomicAdd(pass + tx + (size_t)ty * step, 1u);
      atomicAdd(hit + tx + (size_t)ty * step, 1u);
      my_visits += 2;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) my_visits += __shfl_xor_sync(0xffffffffu, my_visits, d);
  if (lane == 0 && my_visits) atomicAdd(visits, my_visits);
}

// OccupancyGrid::Update / UpdateCell (Karto.h:5953-5990): MinPassThrough = 2, OccupancyThreshold = 0.1
__global__ void k_occ_threshold(const uint32_t *__restrict__ pass, const uint32_t *__restrict__ hit, int n,
                                uint8_t *__restrict__ cells) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t v = 0;
  const uint32_t p = pass[i];
  if (p > 2u) {
    const double ratio = (double)hit[i] / (double)p;
    v = ratio > 0.1 ? (uint8_t)GRID_OCCUPIED : (uint8_t)GRID_FREE;
  }
  cells[i] = v;
}

// SlamKarto::updateMap payload (karto_slam.cc:546-569): unknown -> -1, occupied -> 100, free -> 0; row-major w x h
__global__ void k_occ_ros(const uint8_t *__restrict__ cells, int w, int h, int step, int8_t *__restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const int x = i % w, y = i / w;
  const uint8_t v = cells[x + (size_t)y * step];
  out[i] = v == 0 ? -1 : (v == GRID_OCCUPIED ? 100 : 0);
}

}  // namespace b2s

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
  B2S_CUDA_CHECK(d_ranges.alloc(std::max<size_t>(M * n, 1)));
  B2S_CUDA_CHECK(d_poses.alloc(std::max<size_t>(M * 3, 1)));
  B2S_CUDA_CHECK(d_sensor.alloc(std::max<size_t>(M * 3, 1)));
  B2S_CUDA_CHECK(d_pts.alloc(std::max<size_t>(M * n * 2, 1)));
  B2S_CUDA_CHECK(d_bbox.alloc((M + 1) * 4));
  B2S_CUDA_CHECK(d_visits.alloc(1));
  if (n && M) B2S_CUDA_CHECK(cudaMemcpyAsync(d_ranges, ranges, sizeof(double) * M * n, cudaMemcpyHostToDevice, st));
  if (M) B2S_CUDA_CHECK(cudaMemcpyAsync(d_poses, poses, sizeof(double) * M * 3, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemsetAsync(d_visits, 0, sizeof(unsigned long long), st));
  double bb[4];
  if (M) k_scan_points<<<(unsigned)M, 256, 0, st>>>(d_ranges, d_poses, *laser, d_sensor, d_pts, nullptr, nullptr);
  if (given_bbox) {
    for (int i = 0; i < 4; i++) bb[i] = given_bbox[i];
  } else {
    k_scan_bbox<<<(unsigned)M, 256, 0, st>>>(d_ranges, d_sensor, d_pts, *laser, d_bbox);
    k_bbox_union<<<1, 256, 0, st>>>(d_bbox, n_scans, d_bbox + 4 * M);
    B2S_CUDA_CHECK(cudaGetLastError());
    B2S_CUDA_CHECK(cudaMemcpyAsync(bb, d_bbox + 4 * M, sizeof(bb), cudaMemcpyDeviceToHost, st));
    B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  if (bbox_out) {
    for (int i = 0; i < 4; i++) bbox_out[i] = bb[i];
    return B2S_OK;
  }
  // OccupancyGrid::ComputeDimensions (Karto.h:5816-5821)
  const double scale = 1.0 / resolution;
  b2s_occ_grid_info &I = g->info;
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
    k_raytrace<<<blocks, 256, 0, st>>>(d_ranges, d_sensor, d_pts, *laser, n_beams, I.width, I.height, I.width_step,
                                       I.offset[0], I.offset[1], scale, g->d_pass, g->d_hit, d_visits);
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
