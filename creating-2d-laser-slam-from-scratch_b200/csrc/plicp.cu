// K3 (lesson3) — PL-ICP fine alignment on H100 (sm_90a).  Product code: CUDA only.
//
// Reference call site: reference/lesson3/src/plicp_odometry.cc:285-322 (LaserScanToLDP), :391 (sm_icp),
// :72-185 (sm_params).  The arithmetic of sm_icp lives in CSM, an external library that is not part of the reference
// tree and has no pinned version (PARITY UNPINNED, DESIGN.md §7); this kernel implements the published algorithm
// (A. Censi, "An ICP variant using a point-to-line metric", ICRA 2008) with CSM's loop structure as selected by the
// parameters the reference sets: angular-window nearest-neighbour correspondences with the nearer index-neighbour
// as segment end, duplicate-correspondence pruning (3x rule), percentile / adaptive trimming on point-to-segment
// distances, closed-form point-to-line minimisation (GPC: Lagrange multiplier = largest real root of a quartic).
//
// One CTA per scan pair, the WHOLE iteration loop inside one launch (no host round trips): both scans, the
// transformed scan and the correspondence tables live in shared memory (82 B per beam); every step of an iteration is
// parallel over beams, the trimming percentiles are found by rank counting, the 4x4 system is reduced in a fixed
// order (deterministic).  Batches of independent pairs fill the GPU; a single odometry stream is latency bound.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "plicp_pair.cuh"

using namespace b2s;

namespace b2s {

__global__ void __launch_bounds__(ICP_THREADS)
    k_plicp(b2s_icp_params P, int n, const double *__restrict__ ref_r, const double *__restrict__ sens_r,
            const double *__restrict__ theta, double range_min, double range_max, const double *__restrict__ guess,
            b2s_icp_result *__restrict__ results) {
  extern __shared__ __align__(16) unsigned char icp_smem[];
  __shared__ double red[ICP_THREADS][17];
  __shared__ double xs[8];
  __shared__ int s_cnt[4];
  double *rx, *ry, *sx, *sy;
  uint8_t *rv, *sv;
  IcpPairSmem S;
  icp_carve(icp_smem, n, rx, ry, sx, sy, rv, sv, S);
  S.rx = rx; S.ry = ry; S.sx = sx; S.sy = sy; S.rv = rv; S.sv = sv;
  S.red = red; S.xs = xs; S.s_cnt = s_cnt;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < n; i += ICP_THREADS) {
    const double th = theta[i];
    icp_load_point(ref_r[(size_t)b * n + i], th, range_min, range_max, rx, ry, rv, i);
    icp_load_point(sens_r[(size_t)b * n + i], th, range_min, range_max, sx, sy, sv, i);
  }
  icp_pair(P, n, theta[0], theta[n - 1], S, guess + 3 * b, results + b);
}

}  // namespace b2s

extern "C" b2s_status b2s_plicp_match(const b2s_icp_params *params, int batch, int n, const double *ref_ranges,
                                      const double *sens_ranges, const double *theta, double range_min,
                                      double range_max, const double *first_guess, int device, void *cuda_stream,
                                      b2s_icp_result *results) {
  B2S_NVTX("K3 PL-ICP batch");
  if (!params || !ref_ranges || !sens_ranges || !theta || !first_guess || !results || batch <= 0 || n < 3 ||
      params->max_iterations < 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_match: null/invalid argument");
  if (b2s_status st = open_device(device)) return st;
  // shared memory: the kernel's static arrays + the per-beam dynamic part must fit the opt-in limit of the device
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_plicp));
  int optin = 0;
  B2S_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t smem = (size_t)n * ICP_SMEM_PER_BEAM + 64;
  if (smem + fa.sharedSizeBytes > (size_t)optin) B2S_FAIL(B2S_ERR_TOO_LARGE, "too many beams for the shared-memory PL-ICP kernel");
  // always opt in: static + dynamic crosses the 48 KB default long before the dynamic part alone does
  B2S_CUDA_CHECK(cudaFuncSetAttribute(k_plicp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)optin - fa.sharedSizeBytes)));
  Stream st;  // declared before the buffers freed on it
  B2S_CUDA_CHECK(st.init(cuda_stream));
  const size_t bn = (size_t)batch * n;
  AsyncBuf<double> d_ref(st), d_sens(st), d_theta(st), d_guess(st);
  AsyncBuf<b2s_icp_result> d_res(st);
  B2S_CUDA_CHECK(d_ref.alloc(bn));
  B2S_CUDA_CHECK(d_sens.alloc(bn));
  B2S_CUDA_CHECK(d_theta.alloc(n));
  B2S_CUDA_CHECK(d_guess.alloc(3 * (size_t)batch));
  B2S_CUDA_CHECK(d_res.alloc(batch));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_ref, ref_ranges, sizeof(double) * bn, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_sens, sens_ranges, sizeof(double) * bn, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_theta, theta, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_guess, first_guess, sizeof(double) * 3 * batch, cudaMemcpyHostToDevice, st));
  k_plicp<<<batch, ICP_THREADS, smem, st>>>(*params, n, d_ref, d_sens, d_theta, range_min, range_max, d_guess, d_res);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(results, d_res, sizeof(b2s_icp_result) * batch, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(st));
  return B2S_OK;
}
