// lesson2 — PCL point-to-point ICP between LaserScans on H100 (sm_90a).  Product code: CUDA only.
//
// Reference call site: reference/lesson2/src/scan_match_icp.cc: ConvertScan2PointCloud (:89-130) turns a LaserScan into
// a pcl::PointCloud<PointXYZ>; ScanMatchWithICP (:135-164) aligns the previous cloud (source) to the current one
// (target) with a default-constructed pcl::IterativeClosestPoint<PointXYZ, PointXYZ> and no initial guess.  The ICP
// lives in PCL, third-party code absent from the reference tree (PARITY UNPINNED, DESIGN.md §2 and §4): this file
// restates PCL 1.8's published behaviour with the node's defaults —
//   - exact Euclidean nearest target of every source point (lowest index among equal distances), no rejection beyond
//     max_correspondence_distance, at least 3 correspondences;
//   - the SVD rigid fit in float, for planar points its 2-D closed form: centroids, cross-covariance S,
//     R = [[a, -b], [b, a]] / sqrt(a^2 + b^2) with (a, b) = (Sxx + Syy, Sxy - Syx), t = c_tgt - R c_src;
//   - final = increment * final, the working cloud transformed by each increment;
//   - DefaultConvergenceCriteria: the iteration cap (converged), the increment's cos(angle) and |t|^2 against
//     1 - transformation_epsilon and transformation_epsilon, the absolute (1e-12) and relative MSE change.
// Only + - * / and a correctly rounded sqrt enter the loop; the beam angles use glibc_math.cuh's restatement of the C
// library's sinf / cosf, and the host takes the yaw with the C library's atan2f.
//
// Two kernels.  k_pcl_cloud converts every scan of the batch once (a scan is in two pairs of a recording).  k_pcl_icp is
// one CTA per pair running the WHOLE iteration loop inside one launch: target, source and the transformed source as
// float2 in shared memory with the correspondence of each source point (32 B per beam).  The nearest-neighbour search
// is a brute-force sweep over the target in shared memory — every thread holds up to four source points, so one
// shared load serves four distance tests.  Reductions run in a fixed order (per-thread strided partials, a shuffle tree
// in each warp, a tree over the warps), the order the CPU restatement mirrors.
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "glibc_math.cuh"

using namespace b2s;

namespace {

constexpr int PI_THREADS = 256;  // lanes of every reduction: the restatement uses the same count
constexpr int PI_WARPS = PI_THREADS / 32;
constexpr int PI_PTS = 4;        // source points per thread per sweep of the target

// what the device hands back per pair; the host turns the matrix into (x, y, yaw)
struct PclIcpOut {
  float f[6];  // final transform, rows f00 f01 tx / f10 f11 ty
  int32_t converged, iterations, n_corr, reserved;
  double fitness;
};

// ConvertScan2PointCloud (:96-123) for one scan per CTA: invalid readings stay at (0, 0, 0), or are compacted away
__global__ void __launch_bounds__(PI_THREADS)
    k_pcl_cloud(const float *__restrict__ ranges, int n, float angle_min, float angle_increment, float range_min,
                float range_max, int drop_invalid, bool use_fma, float2 *__restrict__ clouds, int *__restrict__ counts) {
  __shared__ int warp_n[PI_WARPS];
  __shared__ int s_base;
  const int sc = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float *r = ranges + (size_t)sc * n;
  float2 *out = clouds + (size_t)sc * n;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += PI_THREADS) {
    const int i = c0 + tid;
    float2 p = make_float2(0.0f, 0.0f);
    bool valid = false;
    if (i < n) {
      const float range = r[i];
      valid = isfinite(range) && range > range_min && range < range_max;  // :104-109
      if (valid) {
        const float angle = angle_min + (float)(unsigned)i * angle_increment;  // :112, float
        float sn, cs;
        glibc_sincosf(angle, use_fma, &sn, &cs);
        p = make_float2(range * cs, range * sn);
      }
    }
    if (!drop_invalid) {
      if (i < n) out[i] = p;
      continue;
    }
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) warp_n[warp] = __popc(m);
    __syncthreads();
    int off = s_base;
    for (int w = 0; w < warp; w++) off += warp_n[w];
    if (valid) out[off + __popc(m & ((1u << lane) - 1u))] = p;
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < PI_WARPS; w++) s_base += warp_n[w];
    __syncthreads();
  }
  if (tid == 0) counts[sc] = drop_invalid ? s_base : n;
}

template <class T>
__device__ __forceinline__ T warp_tree(T v) {  // lane l += lane l + d, d = 16 .. 1: the sum lands in lane 0
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
  return v;
}

template <class T>
__device__ __forceinline__ T warps_tree(T *w) {  // w[k] += w[k + d], d = PI_WARPS / 2 .. 1 (one thread)
#pragma unroll
  for (int d = PI_WARPS / 2; d > 0; d >>= 1)
    for (int k = 0; k < d; k++) w[k] += w[k + d];
  return w[0];
}

// exact nearest target of PI_PTS query points: squared distance dx*dx + dy*dy in float, the lowest index among equal
// distances; a query with no target at a finite distance (or a NaN placeholder) keeps j = -1
__device__ __forceinline__ void nearest_pts(const float2 *__restrict__ tgt, int nt, const float2 (&q)[PI_PTS],
                                            int (&bj)[PI_PTS], float (&bd)[PI_PTS]) {
#pragma unroll
  for (int k = 0; k < PI_PTS; k++) { bj[k] = -1; bd[k] = INFINITY; }
#pragma unroll 2
  for (int j = 0; j < nt; j++) {
    const float2 t = tgt[j];
#pragma unroll
    for (int k = 0; k < PI_PTS; k++) {
      const float dx = q[k].x - t.x, dy = q[k].y - t.y;
      const float d = dx * dx + dy * dy;
      if (d < bd[k]) { bd[k] = d; bj[k] = j; }
    }
  }
}

__device__ __forceinline__ float2 apply(const float *f, float2 p) {  // transformPointCloud with a planar Matrix4f
  return make_float2((f[0] * p.x + f[1] * p.y) + f[2], (f[3] * p.x + f[4] * p.y) + f[5]);
}

__global__ void __launch_bounds__(PI_THREADS)
    k_pcl_icp(b2s_pcl_icp_params P, double max_d2, int n, const float2 *__restrict__ clouds, const int *__restrict__ counts,
              const int32_t *__restrict__ pairs, const float *__restrict__ guesses, bool use_fma,
              PclIcpOut *__restrict__ out) {
  extern __shared__ __align__(16) unsigned char pi_smem[];
  float2 *tgt = reinterpret_cast<float2 *>(pi_smem), *src = tgt + n, *cur = src + n;
  int *nn = reinterpret_cast<int *>(cur + n);
  float *nd = reinterpret_cast<float *>(nn + n);
  __shared__ float s_f[6];      // final transform
  __shared__ float s_inc[4];    // increment: c, s, tx, ty
  __shared__ float s_cen[4];    // centroids: source x, y, target x, y
  __shared__ float s_wf[5][PI_WARPS];
  __shared__ double s_wd[PI_WARPS];
  __shared__ int s_wi[PI_WARPS];
  __shared__ int s_state[4];    // stop, converged, iterations, correspondences
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int si = pairs ? pairs[2 * b] : b, ti = pairs ? pairs[2 * b + 1] : b + 1;
  const int ns = counts[si], nt = counts[ti];
  const float2 *cs = clouds + (size_t)si * n, *ct = clouds + (size_t)ti * n;
  for (int i = tid; i < ns; i += PI_THREADS) src[i] = cs[i];
  for (int j = tid; j < nt; j += PI_THREADS) tgt[j] = ct[j];
  __shared__ int s_identity;
  if (tid == 0) {
    // final_transformation_ = guess; the source is transformed first only if the guess is not the identity
    float f[6] = {1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f};
    if (guesses) {
      float sn, c;
      glibc_sincosf(guesses[3 * b + 2], use_fma, &sn, &c);
      f[0] = c; f[1] = -sn; f[2] = guesses[3 * b]; f[3] = sn; f[4] = c; f[5] = guesses[3 * b + 1];
    }
    for (int q = 0; q < 6; q++) s_f[q] = f[q];
    s_identity = f[0] == 1.0f && f[1] == 0.0f && f[2] == 0.0f && f[3] == 0.0f && f[4] == 1.0f && f[5] == 0.0f;
    s_state[0] = 0; s_state[1] = 0; s_state[2] = 0; s_state[3] = 0;
  }
  __syncthreads();
  for (int i = tid; i < ns; i += PI_THREADS) cur[i] = s_identity ? src[i] : apply(s_f, src[i]);
  double prev_mse = DBL_MAX;  // thread 0's copy is the one read
  const double rot_thr = 1.0 - P.transformation_epsilon, trans_thr = P.transformation_epsilon;
  for (;;) {
    // ---- correspondences: each thread's points are i = tid (mod PI_THREADS), as in the transform and reductions
    for (int i0 = tid; i0 < ns; i0 += PI_PTS * PI_THREADS) {
      float2 q[PI_PTS];
      int bj[PI_PTS];
      float bd[PI_PTS];
#pragma unroll
      for (int k = 0; k < PI_PTS; k++) {
        const int i = i0 + k * PI_THREADS;
        q[k] = i < ns ? cur[i] : make_float2(NAN, NAN);
      }
      nearest_pts(tgt, nt, q, bj, bd);
#pragma unroll
      for (int k = 0; k < PI_PTS; k++) {
        const int i = i0 + k * PI_THREADS;
        if (i < ns) {
          nn[i] = (bj[k] >= 0 && !((double)bd[k] > max_d2)) ? bj[k] : -1;
          nd[i] = bd[k];
        }
      }
    }
    // ---- centroids
    int cnt = 0;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int i = tid; i < ns; i += PI_THREADS) {
      const int j = nn[i];
      if (j < 0) continue;
      cnt++;
      acc[0] += cur[i].x; acc[1] += cur[i].y;
      acc[2] += tgt[j].x; acc[3] += tgt[j].y;
    }
    cnt = warp_tree(cnt);
#pragma unroll
    for (int q = 0; q < 4; q++) acc[q] = warp_tree(acc[q]);
    if (lane == 0) {
      s_wi[warp] = cnt;
      for (int q = 0; q < 4; q++) s_wf[q][warp] = acc[q];
    }
    __syncthreads();
    if (tid == 0) {
      const int count = warps_tree(s_wi);
      s_state[3] = count;
      if (count < 3) {  // min_number_correspondences_: not converged
        s_state[0] = 1; s_state[1] = 0;
      } else {
        const float inv_n = 1.0f / (float)count;
        for (int q = 0; q < 4; q++) s_cen[q] = warps_tree(s_wf[q]) * inv_n;
      }
    }
    __syncthreads();
    if (s_state[0]) break;
    // ---- cross-covariance S = sum (p - cp)(q - cq)^T and the correspondence MSE
    const float cpx = s_cen[0], cpy = s_cen[1], cqx = s_cen[2], cqy = s_cen[3];
    float S[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    double mse = 0.0;
    for (int i = tid; i < ns; i += PI_THREADS) {
      const int j = nn[i];
      if (j < 0) continue;
      const float px = cur[i].x - cpx, py = cur[i].y - cpy, qx = tgt[j].x - cqx, qy = tgt[j].y - cqy;
      S[0] += px * qx; S[1] += px * qy; S[2] += py * qx; S[3] += py * qy;
      mse += (double)nd[i];
    }
#pragma unroll
    for (int q = 0; q < 4; q++) S[q] = warp_tree(S[q]);
    mse = warp_tree(mse);
    if (lane == 0) {
      for (int q = 0; q < 4; q++) s_wf[q][warp] = S[q];
      s_wd[warp] = mse;
    }
    __syncthreads();
    if (tid == 0) {
      const float sxx = warps_tree(s_wf[0]), sxy = warps_tree(s_wf[1]), syx = warps_tree(s_wf[2]), syy = warps_tree(s_wf[3]);
      const double m = warps_tree(s_wd) / (double)s_state[3];
      const float a = sxx + syy, bb = sxy - syx, h2 = a * a + bb * bb;
      float c = 1.0f, s = 0.0f;
      if (h2 != 0.0f) {
        const float h = sqrtf(h2);
        c = a / h; s = bb / h;
      }
      const float tx = cqx - (c * cpx - s * cpy), ty = cqy - (s * cpx + c * cpy);
      s_inc[0] = c; s_inc[1] = s; s_inc[2] = tx; s_inc[3] = ty;
      const float f0 = s_f[0], f1 = s_f[1], f2 = s_f[2], f3 = s_f[3], f4 = s_f[4], f5 = s_f[5];
      s_f[0] = c * f0 - s * f3; s_f[1] = c * f1 - s * f4; s_f[2] = (c * f2 - s * f5) + tx;
      s_f[3] = s * f0 + c * f3; s_f[4] = s * f1 + c * f4; s_f[5] = (s * f2 + c * f5) + ty;
      const int it = ++s_state[2];
      bool done;
      if (it >= P.max_iterations) {
        done = true;  // failure_after_max_iter_ = false
      } else {
        const double cos_angle = 0.5 * (double)(((c + c) + 1.0f) - 1.0f);
        const double translation_sqr = (double)((tx * tx + ty * ty) + 0.0f * 0.0f);
        done = (cos_angle >= rot_thr && translation_sqr <= trans_thr) || fabs(m - prev_mse) < 1e-12 ||
               fabs(m - prev_mse) / prev_mse < P.euclidean_fitness_epsilon;
        prev_mse = m;
      }
      s_state[0] = done; s_state[1] = done;
    }
    __syncthreads();
    const float c = s_inc[0], s = s_inc[1], tx = s_inc[2], ty = s_inc[3];
    for (int i = tid; i < ns; i += PI_THREADS) {
      const float2 p = cur[i];
      cur[i] = make_float2((c * p.x - s * p.y) + tx, (s * p.x + c * p.y) + ty);
    }
    if (s_state[0]) break;
    __syncthreads();
  }
  // ---- getFitnessScore(): the original source under the final transform, nearest target distance, averaged
  __syncthreads();
  double sum = 0.0;
  int nr = 0;
  for (int i0 = tid; i0 < ns; i0 += PI_PTS * PI_THREADS) {
    float2 q[PI_PTS];
    int bj[PI_PTS];
    float bd[PI_PTS];
#pragma unroll
    for (int k = 0; k < PI_PTS; k++) {
      const int i = i0 + k * PI_THREADS;
      q[k] = i < ns ? apply(s_f, src[i]) : make_float2(NAN, NAN);
    }
    nearest_pts(tgt, nt, q, bj, bd);
#pragma unroll
    for (int k = 0; k < PI_PTS; k++)
      if (i0 + k * PI_THREADS < ns && bj[k] >= 0 && (double)bd[k] <= DBL_MAX) { sum += (double)bd[k]; nr++; }
  }
  sum = warp_tree(sum);
  nr = warp_tree(nr);
  if (lane == 0) { s_wd[warp] = sum; s_wi[warp] = nr; }
  __syncthreads();
  if (tid == 0) {
    const double fit = warps_tree(s_wd);
    const int total = warps_tree(s_wi);
    PclIcpOut &o = out[b];
    for (int q = 0; q < 6; q++) o.f[q] = s_f[q];
    o.converged = s_state[1];
    o.iterations = s_state[2];
    o.n_corr = s_state[3];
    o.reserved = 0;
    o.fitness = total > 0 ? fit / (double)total : DBL_MAX;
  }
}

}  // namespace

extern "C" b2s_status b2s_pcl_icp_align(const b2s_pcl_icp_params *params, int n_scans, int n, const float *ranges,
                                        float angle_min, float angle_increment, float range_min, float range_max,
                                        int n_pairs, const int32_t *pairs, const float *guesses, int device,
                                        void *cuda_stream, b2s_pcl_icp_result *results) {
  B2S_NVTX("lesson2 PCL ICP align (batch)");
  if (!params || !ranges || !results || n_scans < 1 || n < 1 || n_pairs < 0 || params->max_iterations < 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_pcl_icp_align: null/invalid argument");
  if (!pairs && n_pairs != n_scans - 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_pcl_icp_align: without a pair list n_pairs must be n_scans - 1");
  if (pairs)
    for (int p = 0; p < 2 * n_pairs; p++)
      if (pairs[p] < 0 || pairs[p] >= n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_pcl_icp_align: scan index out of range");
  if (b2s_status st = open_device(device)) return st;
  if (n_pairs == 0) return B2S_OK;
  // shared memory: 32 bytes per beam next to the kernel's static arrays, within the device's opt-in limit
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_pcl_icp));
  int optin = 0;
  B2S_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t smem = (size_t)n * (3 * sizeof(float2) + sizeof(int) + sizeof(float));
  if (smem + fa.sharedSizeBytes > (size_t)optin) B2S_FAIL(B2S_ERR_TOO_LARGE, "too many beams for the shared-memory ICP kernel");
  B2S_CUDA_CHECK(raise_dyn_smem(k_pcl_icp, smem));  // above 48 KB only with the opt-in attribute
  static const bool use_fma = glibc_sincosf_variant_of_host() != 0;
  const double max_d2 = params->max_correspondence_distance * params->max_correspondence_distance;
  Stream st;  // declared before the buffers freed on it
  B2S_CUDA_CHECK(st.init(cuda_stream));
  const size_t nr = (size_t)n_scans * n;
  AsyncBuf<float> d_r(st), d_guess(st);
  AsyncBuf<float2> d_cloud(st);
  AsyncBuf<int> d_cnt(st);
  AsyncBuf<int32_t> d_pairs(st);
  AsyncBuf<PclIcpOut> d_out(st);
  B2S_CUDA_CHECK(d_r.alloc(nr));
  B2S_CUDA_CHECK(d_cloud.alloc(nr));
  B2S_CUDA_CHECK(d_cnt.alloc(n_scans));
  B2S_CUDA_CHECK(d_out.alloc(n_pairs));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_r, ranges, sizeof(float) * nr, cudaMemcpyHostToDevice, st));
  if (pairs) {
    B2S_CUDA_CHECK(d_pairs.alloc(2 * (size_t)n_pairs));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_pairs, pairs, sizeof(int32_t) * 2 * n_pairs, cudaMemcpyHostToDevice, st));
  }
  if (guesses) {
    B2S_CUDA_CHECK(d_guess.alloc(3 * (size_t)n_pairs));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_guess, guesses, sizeof(float) * 3 * n_pairs, cudaMemcpyHostToDevice, st));
  }
  k_pcl_cloud<<<n_scans, PI_THREADS, 0, st>>>(d_r, n, angle_min, angle_increment, range_min, range_max,
                                              params->drop_invalid_points != 0, use_fma, d_cloud, d_cnt);
  B2S_CUDA_CHECK(cudaGetLastError());
  k_pcl_icp<<<n_pairs, PI_THREADS, smem, st>>>(*params, max_d2, n, d_cloud, d_cnt, pairs ? d_pairs.p : nullptr,
                                               guesses ? d_guess.p : nullptr, use_fma, d_out);
  B2S_CUDA_CHECK(cudaGetLastError());
  std::vector<PclIcpOut> h(n_pairs);
  B2S_CUDA_CHECK(cudaMemcpyAsync(h.data(), d_out, sizeof(PclIcpOut) * n_pairs, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int p = 0; p < n_pairs; p++) {
    b2s_pcl_icp_result &r = results[p];
    r.x[0] = h[p].f[2];
    r.x[1] = h[p].f[5];
    r.x[2] = atan2f(h[p].f[3], h[p].f[0]);  // pcl::getTranslationAndEulerAngles: yaw = atan2(t(1,0), t(0,0))
    r.converged = h[p].converged;
    r.iterations = h[p].iterations;
    r.n_correspondences = h[p].n_corr;
    r.fitness_score = h[p].fitness;
  }
  return B2S_OK;
}
