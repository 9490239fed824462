// lesson4 make-map nodes over whole recordings on H100 (sm_90a).  Product code: CUDA only.
//
// Reference behaviour (paths relative to reference/lesson4):
//   GMapping::InitParams / ScanCallback / CreateCache / PublishMap / ComputeMap   src/gmapping/gmapping.cc:44-242
//   HectorMapping::InitParams / ScanCallback / ROSLaserScanToDataContainer / PublishMap
//                                                                                src/hector_mapping/hector_mapping.cc:44-211
//   OccGridMapBase::updateByScanJustOnce / updateLineBresenhami / bresenham2D    include/lesson4/hector_mapping/map/
//                                                                                OccGridMapBase.h:175-300
//
// Both nodes build a fresh map from every scan, so scans are independent and a call runs them in chunks: chunk c is
// computed and copied back on stream c % 2, so the copy of one chunk overlaps the kernels of the next.  The beams' unit
// vectors are taken once per call on the host (glibc double cos / sin, as both nodes call them).
//
// GMapping, per chunk of S scans: a scratch map of packed counters per scan (visits in the low 16 bits, n in the high
// 16; a beam adds at most one visit to a cell, and n_ranges <= B2S_NODE_MAPS_MAX_RANGES < 2^16) filled by one warp per
// beam with RED.ADD along the closed-form Bresenham line of k_gm_update (gmapping_grid.cuh), then one thread per
// payload byte finds the storage cell PublishMap writes there last and classifies it.  Before any chunk, one pass over
// every beam of the call finds the first scan whose rays leave the storage, so a refused call writes nothing.
//
// Hector, per chunk: the payload itself is the map.  Because each scan's map is fresh, a cell's published value
// depends only on sets: occupied iff a drawn beam ends there (bresenhamCellOcc un-frees a freed cell exactly:
// (0 + f) - f == 0, and a later free leaves an occupied cell alone), else free iff a drawn beam passes it, else
// unknown.  So the chunk is set to -1, one warp per beam stores 0 along its line (hector_grid.cuh's bresenham2D step),
// and a second pass stores 100 at every drawn beam's end cell.  Plain byte stores, no atomics.
#include <cmath>
#include <cstdio>
#include <vector>

#include "common.cuh"
#include "gmapping_grid.cuh"
#include "hector_grid.cuh"

using namespace b2s;

namespace {

constexpr size_t CHUNK_BYTES = 256u << 20;  // device memory per stream for one chunk's scratch and payloads

// ---- GMapping ----

struct GmGeom {
  double cx, cy, delta, max_range, max_use, occ_thresh;
  int msx, msy, sx2, sy2, width, height;
};

// the first scan with a kept beam whose end cell, or whose laser cell, lies outside the storage (the node asserts)
__global__ void k_gmn_check(const float *__restrict__ ranges, const double *__restrict__ unit, int n_ranges,
                            long long n_beams, GmGeom g, int *__restrict__ first_bad) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_beams) return;
  const int s = (int)(t / n_ranges), i = (int)(t % n_ranges);
  const auto u = [&] { return make_double2(unit[i], unit[n_ranges + i]); };
  const GmRay r = gm_ray((double)ranges[t], u, 0.0, 0.0, g.cx, g.cy, g.delta, g.sx2, g.sy2, g.max_range, g.max_use);
  if (!r.valid) return;
  const int p0x = gm_world2map(0.0, g.cx, g.delta, g.sx2), p0y = gm_world2map(0.0, g.cy, g.delta, g.sy2);
  const bool out0 = p0x < 0 || p0y < 0 || p0x >= g.msx || p0y >= g.msy;
  const bool out1 = r.p1x < 0 || r.p1y < 0 || r.p1x >= g.msx || r.p1y >= g.msy;
  if (out0 || out1) atomicMin(first_bad, s);
}

// ComputeMap of S scans into packed counters [S][msy][msx]: one warp per beam
__global__ void __launch_bounds__(256)
    k_gmn_update(const float *__restrict__ ranges, const double *__restrict__ unit, int n_ranges, int n_scans, GmGeom g,
                 uint32_t *__restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5, n_beams = (long long)n_scans * n_ranges;
  const int p0x = gm_world2map(0.0, g.cx, g.delta, g.sx2), p0y = gm_world2map(0.0, g.cy, g.delta, g.sy2);
  const size_t cells = (size_t)g.msx * g.msy;
  for (long long b = warp0; b < n_beams; b += nwarps) {
    const int s = (int)(b / n_ranges), i = (int)(b % n_ranges);
    const auto u = [&] { return make_double2(unit[i], unit[n_ranges + i]); };
    const GmRay r = gm_ray((double)ranges[b], u, 0.0, 0.0, g.cx, g.cy, g.delta, g.sx2, g.sy2, g.max_range, g.max_use);
    if (!r.valid) continue;
    uint32_t *__restrict__ c = counts + (size_t)s * cells;
    const GmLine L = gm_line(p0x, p0y, r.p1x, r.p1y);
    for (long long k = lane; k <= L.dmaj; k += 32) {
      if (k == L.k_end) continue;  // every cell but the last of the p0 -> p1 list is free (gmapping.cc:227-235)
      const int2 p = gm_line_cell(L, k);
      atomicAdd(c + p.x + (size_t)p.y * g.msx, 1u);
    }
    if (lane == 0 && r.hit) atomicAdd(c + r.p1x + (size_t)r.p1y * g.msx, (1u << 16) | 1u);  // n++, visits++ (:237-241)
  }
}

// PublishMap (gmapping.cc:141-159) of S scans: payload byte (x0, y0) of width W is written by storage cells
// (x0 + k W, y0 - k); the loop runs x outer, so the largest valid k writes last.  No writer: 0.
__global__ void k_gmn_publish(const uint32_t *__restrict__ counts, long long total, GmGeom g,
                              int8_t *__restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const long long wh = (long long)g.width * g.height;
  const int s = (int)(t / wh);
  const long long o = t - (long long)s * wh;
  const int x0 = (int)(o % g.width), y0 = (int)(o / g.width);
  int8_t v = 0;
  if (x0 < g.msx) {
    const int k = min((g.msx - 1 - x0) / g.width, y0);
    if (y0 - k < g.msy) {
      const uint32_t c = counts[(size_t)s * g.msx * g.msy + (size_t)(x0 + k * g.width) + (size_t)(y0 - k) * g.msx];
      v = gm_classify((int32_t)(c >> 16), (int32_t)(c & 0xffffu), g.occ_thresh);
    }
  }
  out[t] = v;
}

// ---- Hector ----

struct HmGeom {
  float range_min, range_lim;  // kept iff range_min < r < range_lim = range_max - 0.1f
  int bx, by, width, height;
};

__device__ __forceinline__ BresenhamLine hmn_line(const HmGeom &g, float r, double ux, double uy) {
  BresenhamLine L;
  L.ok = false;
  if (!(r > g.range_min && r < g.range_lim)) return L;  // hector_mapping.cc:156
  // Eigen::Vector2f(cos(angle) * dist, sin(angle) * dist): double products rounded to float (:159)
  const float px = (float)__dmul_rn(ux, (double)r), py = (float)__dmul_rn(uy, (double)r);
  return bresenham_line(g.bx, g.by, just_once_end_cell(g.bx, g.by, px, py), g.width, g.height);
}

// bresenhamCellFree along every drawn beam of S scans: one warp per beam stores 0
__global__ void __launch_bounds__(256)
    k_hmn_free(const float *__restrict__ ranges, const double *__restrict__ unit, int n_ranges, int n_scans, HmGeom g,
               int8_t *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5, n_beams = (long long)n_scans * n_ranges;
  const long long wh = (long long)g.width * g.height;
  for (long long b = warp0; b < n_beams; b += nwarps) {
    const int s = (int)(b / n_ranges), i = (int)(b % n_ranges);
    const BresenhamLine L = hmn_line(g, ranges[b], unit[i], unit[n_ranges + i]);
    if (!L.ok) continue;
    int8_t *__restrict__ m = out + (size_t)s * wh;
    const int start = L.y0 * g.width + L.x0;
    for (unsigned int k = lane; k < L.da; k += 32) m[bresenham_offset(L, start, k)] = 0;
  }
}

// bresenhamCellOcc at every drawn beam's end cell, after every free store of the chunk: one thread per beam stores 100
__global__ void k_hmn_occ(const float *__restrict__ ranges, const double *__restrict__ unit, int n_ranges,
                          long long n_beams, HmGeom g, int8_t *__restrict__ out) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_beams) return;
  const int s = (int)(b / n_ranges), i = (int)(b % n_ranges);
  const BresenhamLine L = hmn_line(g, ranges[b], unit[i], unit[n_ranges + i]);
  if (L.ok) out[(size_t)s * g.width * g.height + (size_t)L.y1 * g.width + L.x1] = 100;
}

// ---- shared host path ----

b2s_status check_common(const b2s_laser_scan_msg *geometry, const void *params, int n_scans, const float *ranges,
                        const int32_t *out_dims, const int8_t *out_maps, const char *name) {
  if (!geometry || !params || !out_dims || n_scans < 0 || geometry->n_ranges < 0 ||
      (out_maps && n_scans > 0 && !ranges))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(name) + ": null argument or negative count");
  if (geometry->n_ranges > B2S_NODE_MAPS_MAX_RANGES)
    B2S_FAIL(B2S_ERR_TOO_LARGE, std::string(name) + ": more than B2S_NODE_MAPS_MAX_RANGES ranges per scan");
  return B2S_OK;
}

// the node's (unsigned / int) conversion of a double map dimension, refused where it would not be a usable size
bool node_dim(double d, int &out) {
  if (!(d >= 1.0 && d < 2147483648.0)) return false;
  out = (int)d;
  return true;
}

// Runs the chunks of a call.  upload() enqueues the call's inputs on the first stream; chunk(stream, first, count,
// scratch, payload) enqueues one chunk's kernels.  Each stream owns its scratch and payload buffers.
template <class Chunk>
b2s_status run_chunks(cudaStream_t s0, cudaStream_t s1, int n_scans, size_t scratch_per_scan, size_t payload_per_scan,
                      int8_t *out_maps, Chunk chunk) {
  const size_t per_scan = scratch_per_scan + payload_per_scan;
  const int fit = (int)std::max<size_t>(1, std::min<size_t>(CHUNK_BYTES / per_scan, (size_t)n_scans));
  const int S = std::max(1, std::min(fit, ceil_div(n_scans, 2)));
  Event ready;
  B2S_CUDA_CHECK(ready.create(cudaEventDisableTiming));
  B2S_CUDA_CHECK(cudaEventRecord(ready, s0));
  B2S_CUDA_CHECK(cudaStreamWaitEvent(s1, ready, 0));
  const cudaStream_t st[2] = {s0, s1};
  AsyncBuf<uint8_t> scratch0(s0), scratch1(s1), payload0(s0), payload1(s1);
  AsyncBuf<uint8_t> *scratch[2] = {&scratch0, &scratch1}, *payload[2] = {&payload0, &payload1};
  for (int q = 0; q < 2 && q * S < n_scans; q++) {
    if (scratch_per_scan) B2S_CUDA_CHECK(scratch[q]->alloc(scratch_per_scan * S));
    B2S_CUDA_CHECK(payload[q]->alloc(payload_per_scan * S));
  }
  b2s_status status = B2S_OK;
  for (int first = 0, c = 0; first < n_scans && status == B2S_OK; first += S, c++) {
    const int q = c & 1, count = std::min(S, n_scans - first);
    status = [&]() -> b2s_status {
      if (b2s_status e = chunk(st[q], first, count, scratch[q]->p, (int8_t *)payload[q]->p)) return e;
      B2S_CUDA_CHECK(cudaGetLastError());
      B2S_CUDA_CHECK(cudaMemcpyAsync(out_maps + (size_t)first * payload_per_scan, payload[q]->p,
                                     payload_per_scan * count, cudaMemcpyDeviceToHost, st[q]));
      return B2S_OK;
    }();
  }
  // the second stream reads the call's inputs, which are freed on the first: it finishes before the call returns
  const cudaError_t e1 = cudaStreamSynchronize(s1);
  if (status) return status;
  B2S_CUDA_CHECK(e1);
  B2S_CUDA_CHECK(cudaStreamSynchronize(s0));
  return B2S_OK;
}

int beam_blocks(long long n_beams, int device) {  // 8 warps per block, one warp per beam, grid-stride beyond
  return (int)std::max<long long>(1, std::min<long long>((n_beams + 7) / 8, (long long)sm_count(device) * 16));
}

}  // namespace

extern "C" {

b2s_status b2s_gmapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_gmapping_node_params *params,
                                  int n_scans, const float *ranges, int32_t out_dims[2], int8_t *out_maps, int device,
                                  void *cuda_stream) {
  B2S_NVTX("lesson4 GMapping node maps");
  if (b2s_status e = check_common(geometry, params, n_scans, ranges, out_dims, out_maps, "b2s_gmapping_node_maps"))
    return e;
  const b2s_gmapping_node_params &p = *params;
  const float res_f = (float)p.delta;  // map_.info.resolution is float32 (gmapping.cc:69)
  if (!(p.delta > 0) || !std::isfinite(p.delta) || !(res_f > 0) || !std::isfinite(p.xmin) || !std::isfinite(p.ymin) ||
      !std::isfinite(p.xmax) || !std::isfinite(p.ymax) || !(p.xmax > p.xmin) || !(p.ymax > p.ymin))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_gmapping_node_maps: bad map bounds");
  GmGeom g;
  if (!node_dim((p.xmax - p.xmin) / (double)res_f, g.width) || !node_dim((p.ymax - p.ymin) / (double)res_f, g.height))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_gmapping_node_maps: the map's width or height is not a usable size");
  const long long wh = (long long)g.width * g.height;
  if (wh >= (1ll << 31)) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_gmapping_node_maps: a payload of 2^31 bytes or more");
  out_dims[0] = g.width;
  out_dims[1] = g.height;
  // ScanMatcherMap(center, xmin, ymin, xmax, ymax, delta) (gmapping.cc:130-135, map.h:133-140)
  g.cx = (p.xmin + p.xmax) / 2.0;
  g.cy = (p.ymin + p.ymax) / 2.0;
  g.delta = p.delta;
  g.max_range = p.max_range;
  g.max_use = p.max_use_range;
  g.occ_thresh = p.occ_thresh;
  const double xs = std::ceil((p.xmax - p.xmin) / p.delta), ys = std::ceil((p.ymax - p.ymin) / p.delta);
  if (!(xs < 2147483648.0) || !(ys < 2147483648.0) || xs * ys >= (double)(1ll << 40))
    B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_gmapping_node_maps: map storage too large");
  g.msx = ((int)xs >> 5) << 5;
  g.msy = ((int)ys >> 5) << 5;
  g.sx2 = (int)std::round((g.cx - p.xmin) / p.delta);
  g.sy2 = (int)std::round((g.cy - p.ymin) / p.delta);
  if (g.msx <= 0 || g.msy <= 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_gmapping_node_maps: map smaller than one 32-cell patch");
  if (!out_maps) return B2S_OK;
  if (b2s_status st = open_device(device)) return st;
  if (n_scans == 0) return B2S_OK;
  const int n = geometry->n_ranges;
  // CreateCache (gmapping.cc:112-124): the float angle angle_min + i * angle_increment, widened, then cos / sin
  std::vector<double> unit(2 * (size_t)std::max(n, 1));
  for (int i = 0; i < n; i++) {
    const double angle = geometry->angle_min + (float)(unsigned)i * geometry->angle_increment;
    unit[i] = cos(angle);
    unit[n + i] = sin(angle);
  }
  Stream s0, s1;  // declared before the buffers freed on them
  B2S_CUDA_CHECK(s0.init(cuda_stream));
  B2S_CUDA_CHECK(s1.init(nullptr));
  const long long n_beams = (long long)n_scans * n;
  AsyncBuf<float> d_r(s0);
  AsyncBuf<double> d_unit(s0);
  AsyncBuf<int> d_bad(s0);
  B2S_CUDA_CHECK(d_r.alloc(std::max<long long>(n_beams, 1)));
  B2S_CUDA_CHECK(d_unit.alloc(unit.size()));
  B2S_CUDA_CHECK(d_bad.alloc(1));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, sizeof(float) * n_beams, cudaMemcpyHostToDevice, s0));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_unit, unit.data(), sizeof(double) * unit.size(), cudaMemcpyHostToDevice, s0));
  const int none = n_scans;
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_bad, &none, sizeof(int), cudaMemcpyHostToDevice, s0));
  if (n_beams > 0) {
    k_gmn_check<<<ceil_div(n_beams, 256), 256, 0, s0>>>(d_r, d_unit, n, n_beams, g, d_bad);
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  int bad = none;
  B2S_CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, s0));
  B2S_CUDA_CHECK(cudaStreamSynchronize(s0));
  if (bad < n_scans) {
    char msg[160];
    snprintf(msg, sizeof msg, "b2s_gmapping_node_maps: scan %d: a beam leaves the map (the node asserts, map.h:186-191); "
             "nothing was written", bad);
    B2S_FAIL(B2S_ERR_OUT_OF_RANGE, msg);
  }
  const size_t cells = (size_t)g.msx * g.msy;
  const int dev = device;
  return run_chunks(s0, s1, n_scans, cells * sizeof(uint32_t), (size_t)wh, out_maps,
                    [&](cudaStream_t st, int first, int count, uint8_t *scratch, int8_t *payload) -> b2s_status {
                      uint32_t *counts = reinterpret_cast<uint32_t *>(scratch);
                      B2S_CUDA_CHECK(cudaMemsetAsync(counts, 0, cells * sizeof(uint32_t) * count, st));
                      const long long nb = (long long)count * n;
                      if (nb > 0)
                        k_gmn_update<<<beam_blocks(nb, dev), 256, 0, st>>>(d_r.p + (size_t)first * n, d_unit, n, count,
                                                                          g, counts);
                      const long long total = (long long)count * wh;
                      k_gmn_publish<<<ceil_div(total, 256), 256, 0, st>>>(counts, total, g, payload);
                      return B2S_OK;
                    });
}

b2s_status b2s_hector_mapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_hector_mapping_node_params *params,
                                        int n_scans, const float *ranges, int32_t out_dims[2], int8_t *out_maps,
                                        int device, void *cuda_stream) {
  B2S_NVTX("lesson4 Hector node maps");
  if (b2s_status e = check_common(geometry, params, n_scans, ranges, out_dims, out_maps, "b2s_hector_mapping_node_maps"))
    return e;
  const b2s_hector_mapping_node_params &p = *params;
  if (!(p.delta > 0) || !std::isfinite(p.delta) || !std::isfinite(p.xmin) || !std::isfinite(p.ymin) ||
      !std::isfinite(p.xmax) || !std::isfinite(p.ymax))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_mapping_node_maps: bad map bounds");
  HmGeom g;
  // map_size_ = (xmax_ - xmin_) / resolution_ into an Eigen::Vector2i (hector_mapping.cc:57-58)
  if (!node_dim((p.xmax - p.xmin) / (double)p.delta, g.width) || !node_dim((p.ymax - p.ymin) / (double)p.delta, g.height))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_hector_mapping_node_maps: the map's width or height is not a usable size");
  const long long wh = (long long)g.width * g.height;
  if (wh >= (1ll << 31)) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_hector_mapping_node_maps: a payload of 2^31 bytes or more");
  out_dims[0] = g.width;
  out_dims[1] = g.height;
  if (!out_maps) return B2S_OK;
  if (b2s_status st = open_device(device)) return st;
  if (n_scans == 0) return B2S_OK;
  const int n = geometry->n_ranges;
  g.range_min = geometry->range_min;
  g.range_lim = geometry->range_max - 0.1f;  // maxRangeForContainer (:150)
  // scanBeginMapi of mapPose (800, 800, 0) and origo (0, 0) (OccGridMapBase.h:182-191)
  const int2 b0 = begin_cell(cosf(0.0f), sinf(0.0f), 800.0f, 800.0f, 0.0f, 0.0f);
  g.bx = b0.x;
  g.by = b0.y;
  // ROSLaserScanToDataContainer (:144-163): the float angle accumulated beam by beam, the C library's double cos / sin
  std::vector<double> unit(2 * (size_t)std::max(n, 1));
  float angle = geometry->angle_min;
  for (int i = 0; i < n; i++) {
    unit[i] = cos((double)angle);
    unit[n + i] = sin((double)angle);
    angle += geometry->angle_increment;
  }
  Stream s0, s1;  // declared before the buffers freed on them
  B2S_CUDA_CHECK(s0.init(cuda_stream));
  B2S_CUDA_CHECK(s1.init(nullptr));
  const long long n_beams = (long long)n_scans * n;
  AsyncBuf<float> d_r(s0);
  AsyncBuf<double> d_unit(s0);
  B2S_CUDA_CHECK(d_r.alloc(std::max<long long>(n_beams, 1)));
  B2S_CUDA_CHECK(d_unit.alloc(unit.size()));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, sizeof(float) * n_beams, cudaMemcpyHostToDevice, s0));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_unit, unit.data(), sizeof(double) * unit.size(), cudaMemcpyHostToDevice, s0));
  const int dev = device;
  return run_chunks(s0, s1, n_scans, 0, (size_t)wh, out_maps,
                    [&](cudaStream_t st, int first, int count, uint8_t *, int8_t *payload) -> b2s_status {
                      B2S_CUDA_CHECK(cudaMemsetAsync(payload, 0xff, (size_t)wh * count, st));  // memset(-1) (:186)
                      const long long nb = (long long)count * n;
                      if (nb > 0) {
                        const float *r = d_r.p + (size_t)first * n;
                        k_hmn_free<<<beam_blocks(nb, dev), 256, 0, st>>>(r, d_unit, n, count, g, payload);
                        k_hmn_occ<<<ceil_div(nb, 256), 256, 0, st>>>(r, d_unit, n, nb, g, payload);
                      }
                      return B2S_OK;
                    });
}

}  // extern "C"
