// lesson1 — corner-feature extraction from LaserScans on H100 (sm_90a).  Product code: CUDA only.
//
// Reference: reference/lesson1/src/feature_detection.cc, LaserScan::ScanCallback (:77-179).  Per scan of n <= 1500
// ranges:
//   - the finite readings v[0 .. count) in beam order, orig(k) = the beam of v[k] (:93-106);
//   - c_i = d * d for 5 <= i < count - 5, d = v[i-5] + .. + v[i-1] - v[i] * 10 + v[i+1] + .. + v[i+5] left to right in
//     float (:112-124), stored as S[i] = {c_i, i}; every other entry of S keeps its value-initialised {0, 0} (:81);
//   - six sectors s = count * j / 6, e = count * (j + 1) / 6 - 1: std::sort(S + s, S + e) by value (S[e] is NOT
//     sorted), then a walk from k = e down to s picks the first 20 entries with value > edge_threshold (:139-171);
//   - a picked entry publishes ranges[orig(index)], every other beam 0 (:136, :163).
// One CTA per scan, the scan in shared memory (27 KB at 1 500 beams).  Finite readings are compacted by warp ballot
// and a block-wide scan; the stencil is one thread per i with every add and multiply rounded explicitly, so the build's
// contraction flags cannot change it.  The selection is one warp per sector.  Which entries the node picks depends on
// std::sort's order only when the cut is tied: K = 20 picks (19 if S[e] itself qualifies) come from the sorted range,
// and if the K-th and (K+1)-th largest qualifying values differ, the picked set is simply the entries of rank < K,
// found by rank counting.  When they are equal, one lane sorts the sector with the restated libstdc++ introsort
// (introsort.cuh) and walks it exactly as the node does.  A scan with a NaN curvature (finite ranges of magnitude
// around 1e37 whose stencil overflows both ways) is reported, not sorted: std::sort's order is undefined there.
#include <cmath>

#include "common.cuh"
#include "introsort.cuh"

using namespace b2s;

namespace {

constexpr int FD_THREADS = 256;
constexpr int FD_WARPS = FD_THREADS / 32;
constexpr int FD_MAX = B2S_FEATURE_MAX_BEAMS;  // max_scan_count (:23)
constexpr int FD_SECTORS = 6;
constexpr int FD_PICKS = 20;                   // largestPickedNum <= 20 (:161)
constexpr int FD_MAX_PER_LANE = 32;            // sector entries a lane holds in the rank pass: 32 * 32 > FD_MAX / 6
static_assert(FD_SECTORS <= FD_WARPS, "one warp per sector");
static_assert(FD_MAX / FD_SECTORS <= 32 * FD_MAX_PER_LANE, "the rank pass keeps one bit per entry of a lane");

struct Smooth {  // smoothness_t (:25-29)
  float value;
  int index;
};

// :114-121, left to right, each operation rounded to nearest
__device__ __forceinline__ float curvature(const float *v, int i) {
  float d = __fadd_rn(v[i - 5], v[i - 4]);
  d = __fadd_rn(d, v[i - 3]);
  d = __fadd_rn(d, v[i - 2]);
  d = __fadd_rn(d, v[i - 1]);
  d = __fsub_rn(d, __fmul_rn(v[i], 10.0f));
  d = __fadd_rn(d, v[i + 1]);
  d = __fadd_rn(d, v[i + 2]);
  d = __fadd_rn(d, v[i + 3]);
  d = __fadd_rn(d, v[i + 4]);
  d = __fadd_rn(d, v[i + 5]);
  return __fmul_rn(d, d);
}

__global__ void __launch_bounds__(FD_THREADS)
    k_feature_detect(int n, const float *__restrict__ ranges, float thr, float *__restrict__ out_ranges,
                     int32_t *__restrict__ out_count, float *__restrict__ out_curvature) {
  __shared__ float s_r[FD_MAX];      // the scan; then the curvature row; then the output row
  __shared__ float s_v[FD_MAX];      // new_scan: the finite readings
  __shared__ short s_orig[FD_MAX];   // map_index
  __shared__ Smooth s_S[FD_MAX];     // scan_smoothness_
  __shared__ int s_wn[FD_WARPS];
  __shared__ int s_picks[FD_SECTORS];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float *r = ranges + (size_t)b * n;
  for (int i = tid; i < n; i += FD_THREADS) s_r[i] = r[i];
  __syncthreads();
  // ---- :93-106 compaction of the finite readings, in beam order
  int count = 0;
  for (int c0 = 0; c0 < n; c0 += FD_THREADS) {
    const int i = c0 + tid;
    const bool ok = i < n && isfinite(s_r[i]);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_wn[warp] = __popc(m);
    __syncthreads();
    int off = count;
    for (int w = 0; w < FD_WARPS; w++) {
      if (w < warp) off += s_wn[w];
      count += s_wn[w];
    }
    if (ok) {
      const int k = off + __popc(m & ((1u << lane) - 1u));
      s_v[k] = s_r[i];
      s_orig[k] = (short)i;
    }
    __syncthreads();
  }
  // ---- :112-124 the stencil; the curvature row is NaN wherever it computed nothing.  Every NaN in it is the one
  // quiet NaN 0x7fc00000, so the row does not depend on which NaN an overflowing stencil happens to produce
  const float qnan = __int_as_float(0x7fc00000);
  for (int i = tid; i < n; i += FD_THREADS) s_r[i] = qnan;
  __syncthreads();
  bool nan = false;
  for (int i = tid; i < count; i += FD_THREADS) {
    Smooth sm = {0.0f, 0};
    if (i >= 5 && i < count - 5) {
      const float c = curvature(s_v, i);
      sm.value = c;
      sm.index = i;
      s_r[s_orig[i]] = isnan(c) ? qnan : c;
      nan = nan || isnan(c);
    }
    s_S[i] = sm;
  }
  const bool any_nan = __syncthreads_or(nan);
  float *outr = out_ranges + (size_t)b * n;
  if (out_curvature) {
    float *oc = out_curvature + (size_t)b * n;
    for (int i = tid; i < n; i += FD_THREADS) oc[i] = s_r[i];
  }
  __syncthreads();
  for (int i = tid; i < n; i += FD_THREADS) s_r[i] = 0.0f;  // corner_scan.ranges (:136)
  __syncthreads();
  // ---- :139-171 one warp per sector
  if (!any_nan && warp < FD_SECTORS) {
    const int j = warp;
    const int s = count * j / 6, e = count * (j + 1) / 6 - 1;
    int picks = 0;
    if (s < e) {
      const bool qe = s_S[e].value > thr;  // S[e] is walked first, unsorted
      const int K = qe ? FD_PICKS - 1 : FD_PICKS;
      int q = 0;
      for (int k = s + lane; k < e; k += 32) q += s_S[k].value > thr;
      q = __reduce_add_sync(0xffffffffu, q);
      // rank of each qualifying entry among the sector's values: above the cut when fewer than K values exceed it;
      // the cut is tied when an entry has fewer than K values above it but more than K at or above it
      unsigned in = 0u;
      bool tied = false;
      int it = 0;
      for (int k = s + lane; k < e; k += 32, it++) {
        const float x = s_S[k].value;
        if (!(x > thr)) continue;
        if (q <= K) {
          in |= 1u << it;
          continue;
        }
        int gt = 0, ge = 0;
        for (int t = s; t < e; t++) {
          const float y = s_S[t].value;
          gt += y > x;
          ge += y >= x;
        }
        if (gt < K) in |= 1u << it;
        tied = tied || (gt < K && ge > K);
      }
      if (!__any_sync(0xffffffffu, tied)) {
        if (qe && lane == 0) {
          const int idx = s_S[e].index;
          s_r[s_orig[idx]] = s_v[idx];
        }
        it = 0;
        for (int k = s + lane; k < e; k += 32, it++)
          if (in >> it & 1u) {
            const int idx = s_S[k].index;
            s_r[s_orig[idx]] = s_v[idx];
          }
        picks = min(q + (int)qe, FD_PICKS);
      } else if (lane == 0) {
        introsort(s_S + s, s_S + e);  // std::sort(begin + s, begin + e, by_value()) (:149-150)
        for (int k = e; k >= s; k--) {
          if (s_S[k].value > thr) {
            if (++picks > FD_PICKS) {
              picks = FD_PICKS;
              break;
            }
            const int idx = s_S[k].index;
            s_r[s_orig[idx]] = s_v[idx];
          }
        }
      }
    }
    if (lane == 0) s_picks[j] = picks;
  }
  __syncthreads();
  for (int i = tid; i < n; i += FD_THREADS) outr[i] = s_r[i];
  if (tid == 0 && out_count) {
    int total = 0;
    for (int j = 0; j < FD_SECTORS; j++) total += s_picks[j];
    out_count[b] = any_nan ? -1 : total;
  }
}

}  // namespace

extern "C" b2s_status b2s_feature_detect(int batch, int n, const float *ranges, float edge_threshold, float *out_ranges,
                                         int32_t *out_count, float *out_curvature, int device, void *cuda_stream) {
  B2S_NVTX("lesson1 feature detection (batch)");
  if (!ranges || !out_ranges || batch < 0 || n < 0 || !(edge_threshold >= 0.0f))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_feature_detect: null/invalid argument (edge_threshold must be >= 0)");
  if (n > B2S_FEATURE_MAX_BEAMS) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_feature_detect: more than 1500 beams per scan");
  if (b2s_status st = open_device(device)) return st;
  if (batch == 0) return B2S_OK;
  if (n == 0) {  // no readings, no picks
    if (out_count)
      for (int b = 0; b < batch; b++) out_count[b] = 0;
    return B2S_OK;
  }
  Stream st;  // declared before the buffers freed on it
  B2S_CUDA_CHECK(st.init(cuda_stream));
  const size_t nr = (size_t)batch * n;
  AsyncBuf<float> d_r(st), d_out(st), d_curv(st);
  AsyncBuf<int32_t> d_cnt(st);
  B2S_CUDA_CHECK(d_r.alloc(nr));
  B2S_CUDA_CHECK(d_out.alloc(nr));
  if (out_count) B2S_CUDA_CHECK(d_cnt.alloc(batch));
  if (out_curvature) B2S_CUDA_CHECK(d_curv.alloc(nr));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, sizeof(float) * nr, cudaMemcpyHostToDevice, st));
  k_feature_detect<<<batch, FD_THREADS, 0, st>>>(n, d_r, edge_threshold, d_out, out_count ? d_cnt.p : nullptr,
                                                 out_curvature ? d_curv.p : nullptr);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out_ranges, d_out, sizeof(float) * nr, cudaMemcpyDeviceToHost, st));
  if (out_count)
    B2S_CUDA_CHECK(cudaMemcpyAsync(out_count, d_cnt, sizeof(int32_t) * batch, cudaMemcpyDeviceToHost, st));
  if (out_curvature)
    B2S_CUDA_CHECK(cudaMemcpyAsync(out_curvature, d_curv, sizeof(float) * nr, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  return B2S_OK;
}
