// K2b — lesson4 GMapping hit/visit map update on H100 (sm_90a).  Product code: CUDA only.
//
// Reference behaviour (paths relative to reference/lesson4):
//   GMapping::ComputeMap / PublishMap                 src/gmapping/gmapping.cc:127-242
//   GridLineTraversal::gridLineCore / gridLine        include/lesson4/gmapping/grid/gridlinetraversal.h:27-207
//   Map ctor (32-cell patch rounding), world2map      include/lesson4/gmapping/grid/map.h:133-140, 171-174
//   PointAccumulator::update / operator double        include/lesson4/gmapping/grid/map.h:27, 37-48
//
// One warp per beam, lanes over the steps of the midpoint Bresenham line, whose decision variable has the closed
// form  j(k) = floor((2*k*dmin + dmaj) / (2*dmaj))  (k = steps from the end with the smaller dominant coordinate).
// All line cells except the beam's end cell get visits++ (RED.ADD); a hit adds n++, visits++ and the float hit
// position (atomicAdd float: the only non-integer state; its summation order is not the reference's, so acc agrees
// to float rounding only — the counters are bit-exact).
// HBM layout: n[sizeY][sizeX] i32, visits[...] i32, acc_x / acc_y [...] f32 (dense; the reference's 32x32 patch
// hierarchy is a CPU allocation detail, the published map is dense).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "gmapping_grid.cuh"

using namespace b2s;

struct b2s_gmap {
  Stream stream;
  int device = 0;
  double cx = 0, cy = 0, delta = 0, xmin = 0, ymin = 0, xmax = 0, ymax = 0;
  int msx = 0, msy = 0, sx2 = 0, sy2 = 0;
  Buf<int32_t> d_n, d_visits;
  Buf<float> d_accx, d_accy;
  Buf<int> d_flag;
  Buf<double> d_in;     // [2][capacity]: ranges, angles of the current scan
  HostBuf<double> h_in;  // pinned staging of the same
  HostBuf<int> h_flag;
};

namespace b2s {

// any ray leaving the map? (the reference asserts / indexes out of range there: map.h:186-191, harray2d.h:206-227)
__global__ void k_gm_check(const double *__restrict__ ranges, const double *__restrict__ angles, int nb, double lx,
                           double ly, double cx, double cy, double delta, int sx2, int sy2, int msx, int msy,
                           double max_range, double max_use, int *__restrict__ flag) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  const auto u = [&] { return make_double2(cos(angles[i]), sin(angles[i])); };
  GmRay r = gm_ray(ranges[i], u, lx, ly, cx, cy, delta, sx2, sy2, max_range, max_use);
  if (r.valid && (r.p1x < 0 || r.p1y < 0 || r.p1x >= msx || r.p1y >= msy)) *flag = 1;
}

__global__ void __launch_bounds__(256)
    k_gm_update(const double *__restrict__ ranges, const double *__restrict__ angles, int nb, double lx, double ly,
                double cx, double cy, double delta, int sx2, int sy2, int msx, double max_range, double max_use,
                int32_t *__restrict__ n, int32_t *__restrict__ visits, float *__restrict__ accx,
                float *__restrict__ accy, const int *__restrict__ leaves_map) {
  if (*leaves_map) return;  // k_gm_check found a beam leaving the map: the reference asserts, nothing may be updated
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int p0x = gm_world2map(lx, cx, delta, sx2), p0y = gm_world2map(ly, cy, delta, sy2);
  for (int i = warp0; i < nb; i += nwarps) {
    const auto u = [&] { return make_double2(cos(angles[i]), sin(angles[i])); };
    GmRay r = gm_ray(ranges[i], u, lx, ly, cx, cy, delta, sx2, sy2, max_range, max_use);
    if (!r.valid) continue;
    const GmLine L = gm_line(p0x, p0y, r.p1x, r.p1y);
    for (long long k = lane; k <= L.dmaj; k += 32) {
      if (k == L.k_end) continue;  // all points but the last of the p0 -> p1 list are free (gmapping.cc:229-235)
      const int2 c = gm_line_cell(L, k);
      atomicAdd(visits + c.x + (size_t)c.y * msx, 1);
    }
    if (lane == 0 && r.hit) {  // gmapping.cc:237-241, map.h:37-48
      const size_t c = (size_t)r.p1x + (size_t)r.p1y * msx;
      atomicAdd(accx + c, (float)r.hx);
      atomicAdd(accy + c, (float)r.hy);
      atomicAdd(n + c, 1);
      atomicAdd(visits + c, 1);
    }
  }
}

// GMapping::PublishMap thresholding (gmapping.cc:141-159) into width x height (MAP_IDX = width*y + x).  One thread per
// published byte.  Storage cells (x + k*width, y - k) all land on byte (x, y); the reference loops x outer, y inner,
// so the one with the largest x is written last and wins.  msx <= width + 1, so only storage cell (width, y - 1) can
// shadow (0, y).  A byte no storage cell maps to keeps the caller's 0.
__global__ void k_gm_ros(const int32_t *__restrict__ n, const int32_t *__restrict__ visits, int msx, int msy,
                         double occ_thresh, int width, int height, int8_t *__restrict__ out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)width * height) return;
  int x = (int)(o % width), y = (int)(o / width);
  if (x == 0 && y > 0 && width < msx && y - 1 < msy) { x = width; y -= 1; }
  if (x >= msx || y >= msy) return;
  const size_t c = (size_t)x + (size_t)y * msx;
  out[o] = gm_classify(n[c], visits[c], occ_thresh);
}

}  // namespace b2s

extern "C" void b2s_gmap_destroy(b2s_gmap *g);
extern "C" {

b2s_status b2s_gmap_create(double center_x, double center_y, double xmin, double ymin, double xmax, double ymax,
                           double delta, int device, void *cuda_stream, b2s_gmap **out) {
  if (!out || !(delta > 0) || !(xmax > xmin) || !(ymax > ymin)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_gmap_create: bad map bounds");
  *out = nullptr;
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<b2s_gmap, decltype(&b2s_gmap_destroy)> g(new (std::nothrow) b2s_gmap(), b2s_gmap_destroy);
  if (!g) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  g->device = device;
  g->cx = center_x; g->cy = center_y; g->delta = delta;
  g->xmin = xmin; g->ymin = ymin; g->xmax = xmax; g->ymax = ymax;
  const int xs = (int)ceil((xmax - xmin) / delta), ys = (int)ceil((ymax - ymin) / delta);  // map.h:133
  g->msx = (xs >> 5) << 5;  // HierarchicalArray2D(xsize >> 5 patches) << patch magnitude (harray2d.h:75-80)
  g->msy = (ys >> 5) << 5;
  g->sx2 = (int)round((center_x - xmin) / delta);  // map.h:139-140
  g->sy2 = (int)round((center_y - ymin) / delta);
  if (g->msx <= 0 || g->msy <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map smaller than one 32-cell patch");
  B2S_CUDA_CHECK(g->stream.init(cuda_stream));
  const size_t cells = (size_t)g->msx * g->msy;
  B2S_CUDA_CHECK(g->d_n.reserve(cells));
  B2S_CUDA_CHECK(g->d_visits.reserve(cells));
  B2S_CUDA_CHECK(g->d_accx.reserve(cells));
  B2S_CUDA_CHECK(g->d_accy.reserve(cells));
  B2S_CUDA_CHECK(g->d_flag.reserve(1));
  for (void *p : {(void *)g->d_n, (void *)g->d_visits, (void *)g->d_accx, (void *)g->d_accy})
    B2S_CUDA_CHECK(cudaMemsetAsync(p, 0, cells * 4, g->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  *out = g.release();
  return B2S_OK;
}

void b2s_gmap_destroy(b2s_gmap *g) {
  if (!g) return;
  cudaSetDevice(g->device);
  cudaStreamSynchronize(g->stream);
  delete g;
}

b2s_status b2s_gmap_size(const b2s_gmap *g, int32_t size_xy[2]) {
  if (!g || !size_xy) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  size_xy[0] = g->msx;
  size_xy[1] = g->msy;
  return B2S_OK;
}

b2s_status b2s_gmap_compute_map(b2s_gmap *g, const double *ranges, const double *angles, int n,
                                const double laser_pose[3], double max_range, double max_urange) {
  B2S_NVTX("K2b ComputeMap");
  if (!g || !ranges || !angles || !laser_pose || n < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (n == 0) return B2S_OK;
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  cudaStream_t st = g->stream;
  const double lx = laser_pose[0], ly = laser_pose[1];  // ComputeMap uses lp = (x, y, 0): beam angles are absolute
  const int p0x = cast_i32(round((lx - g->cx) / g->delta)) + g->sx2, p0y = cast_i32(round((ly - g->cy) / g->delta)) + g->sy2;
  if (p0x < 0 || p0y < 0 || p0x >= g->msx || p0y >= g->msy) B2S_FAIL(B2S_ERR_OUT_OF_RANGE, "laser position outside the map");
  // scan buffers live in the handle: no per-call allocation
  B2S_CUDA_CHECK(g->d_in.reserve(2 * (size_t)std::max(n, 2048)));
  B2S_CUDA_CHECK(g->h_in.reserve(2 * (size_t)std::max(n, 2048)));
  B2S_CUDA_CHECK(g->h_flag.reserve(1));
  std::memcpy(g->h_in, ranges, sizeof(double) * n);
  std::memcpy(g->h_in + n, angles, sizeof(double) * n);
  double *d_r = g->d_in, *d_a = g->d_in + n;
  B2S_CUDA_CHECK(cudaMemcpyAsync(g->d_in, g->h_in, sizeof(double) * 2 * (size_t)n, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemsetAsync(g->d_flag, 0, sizeof(int), st));
  k_gm_check<<<ceil_div(n, 256), 256, 0, st>>>(d_r, d_a, n, lx, ly, g->cx, g->cy, g->delta, g->sx2, g->sy2, g->msx,
                                               g->msy, max_range, max_urange, g->d_flag);
  // the update reads the verdict on the device (no host round trip between check and update)
  k_gm_update<<<std::min(ceil_div(n, 8), sm_count(g->device) * 8), 256, 0, st>>>(d_r, d_a, n, lx, ly, g->cx, g->cy, g->delta, g->sx2,
                                                                g->sy2, g->msx, max_range, max_urange, g->d_n,
                                                                g->d_visits, g->d_accx, g->d_accy, g->d_flag);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(g->h_flag, g->d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  if (*g->h_flag) {
    set_last_error("a beam leaves the map (the reference asserts here, map.h:186-191); nothing was updated");
    return B2S_ERR_OUT_OF_RANGE;
  }
  return B2S_OK;
}

b2s_status b2s_gmap_copy(b2s_gmap *g, int32_t *n, int32_t *visits, float *acc_x, float *acc_y) {
  if (!g) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  const size_t bytes = (size_t)g->msx * g->msy * 4;
  if (n) B2S_CUDA_CHECK(cudaMemcpyAsync(n, g->d_n, bytes, cudaMemcpyDeviceToHost, g->stream));
  if (visits) B2S_CUDA_CHECK(cudaMemcpyAsync(visits, g->d_visits, bytes, cudaMemcpyDeviceToHost, g->stream));
  if (acc_x) B2S_CUDA_CHECK(cudaMemcpyAsync(acc_x, g->d_accx, bytes, cudaMemcpyDeviceToHost, g->stream));
  if (acc_y) B2S_CUDA_CHECK(cudaMemcpyAsync(acc_y, g->d_accy, bytes, cudaMemcpyDeviceToHost, g->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

b2s_status b2s_gmap_copy_ros(b2s_gmap *g, int8_t *out) {
  if (!g || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(g->device));
  // map_.info.width/height = (xmax - xmin) / resolution truncated to uint32 (gmapping.cc:70-71)
  const int width = (int)(uint32_t)((g->xmax - g->xmin) / g->delta), height = (int)(uint32_t)((g->ymax - g->ymin) / g->delta);
  if (width <= 0 || height <= 0) return B2S_OK;
  AsyncBuf<int8_t> d(g->stream);
  B2S_CUDA_CHECK(d.alloc((size_t)width * height));
  B2S_CUDA_CHECK(cudaMemsetAsync(d, 0, (size_t)width * height, g->stream));
  k_gm_ros<<<ceil_div((long long)width * height, 256), 256, 0, g->stream>>>(g->d_n, g->d_visits, g->msx, g->msy, 0.25,
                                                                          width, height, d);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, d, (size_t)width * height, cudaMemcpyDeviceToHost, g->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(g->stream));
  return B2S_OK;
}

}  // extern "C"
