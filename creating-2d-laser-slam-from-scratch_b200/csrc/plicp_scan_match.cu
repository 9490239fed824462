// K3 (lesson3) — the scan-to-scan PL-ICP node on H100 (sm_90a): ScanMatchPLICP::ScanCallback
// (reference/lesson3/src/scan_match_plicp.cc:162-300) for B independent recordings, each of its own laser, every scan
// pair of every recording in ONE launch.
//
// The node matches each scan against the scan before it from a zero first guess, so the pairs of a recording do not
// depend on each other: one CTA per scan pair, spread over every SM even for a single recording.  The CTA converts both
// scans from their float32 ranges into the two slots of the pair kernel's shared memory (LaserScanToLDP, :220-261, each
// scan with its own message's range fields) and runs the pair matcher (plicp_pair.cuh, the code of b2s_plicp_match).
// A recording's first scan of a call is matched against the last scan of its previous call, kept in device memory with
// its range fields; a second, stream-ordered kernel refreshes that store after the pair kernel has read it, so calls
// over consecutive parts of a recording equal one call.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "plicp_pair.cuh"

using namespace b2s;

namespace b2s {

// LaserScanToLDP's beam angle (:243): angle_min + i * angle_increment summed in float, then widened
__device__ __forceinline__ double sm_beam_theta(float angle_min, float angle_increment, int i) {
  return (double)__fadd_rn(angle_min, __fmul_rn((float)i, angle_increment));
}

struct ScanMatchLaunch {
  b2s_icp_params P;
  int batch;
  const int32_t *n_beams;          // [B]
  const float *angle_min;          // [B]
  const float *angle_increment;    // [B]
  const long long *first;          // [B + 1]: index of recording b's first scan of this call in limits / out
  const long long *range_off;      // [B]: offset of recording b's first scan of this call in ranges
  const long long *store_off;      // [B]: offset of recording b's last scan in store_ranges
  const float *ranges;             // [sum over b of n_scans[b] * n_beams[b]]
  const float *limits;             // [sum][2]: range_min, range_max of every scan
  const float *store_ranges;       // [sum n_beams]: every recording's last scan (persistent)
  const float *store_limits;       // [B][2]: its range fields (persistent)
  const int32_t *seen;             // [B]: 1 once the recording has a last scan (persistent)
  b2s_plicp_scan_match_step *out;  // [sum]
};

__global__ void __launch_bounds__(ICP_THREADS) k_plicp_scan_match(ScanMatchLaunch A) {
  extern __shared__ __align__(16) unsigned char icp_smem[];
  __shared__ double red[ICP_THREADS][17];
  __shared__ double xs[8];
  __shared__ int s_cnt[4];
  const long long g = blockIdx.x;
  // the recording of scan g: the last b with first[b] <= g (recordings with no scan in this call have first[b] ==
  // first[b + 1] and are skipped by taking the last such b)
  int lo = 0, hi = A.batch - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (A.first[mid] <= g) lo = mid; else hi = mid - 1;
  }
  const int b = lo, tid = threadIdx.x, n = A.n_beams[b];
  const long long s = g - A.first[b];
  b2s_plicp_scan_match_step *o = A.out + g;
  if (s == 0 && !A.seen[b]) {
    // the scan that initialises the node (:165-175): it only becomes the previous scan
    if (tid == 0) *o = b2s_plicp_scan_match_step{};
    return;
  }
  double *rx, *ry, *cx, *cy;  // previous scan slot, current scan slot
  uint8_t *rv, *cv;
  IcpPairSmem S;
  icp_carve(icp_smem, n, rx, ry, cx, cy, rv, cv, S);
  S.rx = rx; S.ry = ry; S.rv = rv; S.sx = cx; S.sy = cy; S.sv = cv;
  S.red = red; S.xs = xs; S.s_cnt = s_cnt;
  const float amin = A.angle_min[b], ainc = A.angle_increment[b];
  const float *cur = A.ranges + A.range_off[b] + s * n;
  const float *prev = s == 0 ? A.store_ranges + A.store_off[b] : cur - n;
  const float *cl = A.limits + 2 * g;
  const float *pl = s == 0 ? A.store_limits + 2 * b : cl - 2;
  // double r compared against the message's float fields (:229-231): NaN and +-inf are never inside the window
  const double pmin = pl[0], pmax = pl[1], cmin = cl[0], cmax = cl[1];
  for (int i = tid; i < n; i += ICP_THREADS) {
    const double th = sm_beam_theta(amin, ainc, i);
    icp_load_point(prev[i], th, pmin, pmax, rx, ry, rv, i);
    icp_load_point(cur[i], th, cmin, cmax, cx, cy, cv, i);
  }
  // ScanMatchWithPLICP (:266-300): sm_icp from a zero first guess, min_theta / max_theta = theta[0] / theta[n - 1]
  const double guess[3] = {0.0, 0.0, 0.0};
  b2s_icp_result res;
  icp_pair(A.P, n, sm_beam_theta(amin, ainc, 0), sm_beam_theta(amin, ainc, n - 1), S, guess, &res);
  if (tid == 0) {
    b2s_plicp_scan_match_step z = {};
    z.icp = res;
    z.theta_deg = res.x[2] * 180 / M_PI;  // what the node prints (:289), in its operation order
    z.matched = 1;
    *o = z;
  }
}

// After the pair kernel: every recording with a scan in this call keeps its last one and that scan's range fields.
__global__ void k_plicp_scan_match_store(ScanMatchLaunch A, float *store_ranges, float *store_limits, int32_t *seen) {
  const int b = blockIdx.x;
  const long long cnt = A.first[b + 1] - A.first[b];
  if (cnt == 0) return;
  const int n = A.n_beams[b];
  const float *last = A.ranges + A.range_off[b] + (cnt - 1) * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) store_ranges[A.store_off[b] + i] = last[i];
  if (threadIdx.x == 0) {
    const long long g = A.first[b + 1] - 1;
    store_limits[2 * b] = A.limits[2 * g];
    store_limits[2 * b + 1] = A.limits[2 * g + 1];
    seen[b] = 1;
  }
}

}  // namespace b2s

struct b2s_plicp_scan_match {
  Stream st;  // declared first: destroyed after the buffers
  int device = 0, batch = 0;
  b2s_icp_params params;
  std::vector<int32_t> n_beams;
  std::vector<long long> store_off;
  Buf<int32_t> d_n_beams, seen;
  Buf<float> d_angle_min, d_angle_increment, store_ranges, store_limits, ranges, limits;
  Buf<long long> d_store_off, first, range_off;
  Buf<b2s_plicp_scan_match_step> out;
};

// the pair kernel's dynamic shared memory for n beams
static size_t scan_match_smem(int n) { return (size_t)n * ICP_SMEM_PER_BEAM + 64; }

extern "C" b2s_status b2s_plicp_scan_match_create(const b2s_icp_params *params, int batch, const int32_t *n_beams,
                                                  const float *angle_min, const float *angle_increment, int device,
                                                  void *cuda_stream, b2s_plicp_scan_match **out) {
  B2S_NVTX("K3 PL-ICP scan match create");
  if (!params || !out || batch <= 0 || !n_beams || !angle_min || !angle_increment || params->max_iterations < 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_create: null/invalid argument");
  int max_n = 0;
  for (int b = 0; b < batch; b++) {
    if (n_beams[b] < 3) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_create: fewer than 3 beams");
    max_n = std::max(max_n, (int)n_beams[b]);
  }
  *out = nullptr;
  if (b2s_status s = open_device(device)) return s;
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_plicp_scan_match));
  int optin = 0;
  B2S_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  if (scan_match_smem(max_n) + fa.sharedSizeBytes > (size_t)optin)
    B2S_FAIL(B2S_ERR_TOO_LARGE, "too many beams for the shared-memory PL-ICP kernel");
  B2S_CUDA_CHECK(raise_dyn_smem(k_plicp_scan_match, scan_match_smem(max_n)));
  std::unique_ptr<b2s_plicp_scan_match> h(new b2s_plicp_scan_match());
  B2S_CUDA_CHECK(h->st.init(cuda_stream));
  h->device = device; h->batch = batch; h->params = *params;
  h->n_beams.assign(n_beams, n_beams + batch);
  h->store_off.resize(batch);
  long long total_beams = 0;
  for (int b = 0; b < batch; b++) {
    h->store_off[b] = total_beams;
    total_beams += n_beams[b];
  }
  B2S_CUDA_CHECK(h->d_n_beams.reserve(batch));
  B2S_CUDA_CHECK(h->d_angle_min.reserve(batch));
  B2S_CUDA_CHECK(h->d_angle_increment.reserve(batch));
  B2S_CUDA_CHECK(h->d_store_off.reserve(batch));
  B2S_CUDA_CHECK(h->seen.reserve(batch));
  B2S_CUDA_CHECK(h->store_ranges.reserve((size_t)total_beams));
  B2S_CUDA_CHECK(h->store_limits.reserve(2 * (size_t)batch));
  B2S_CUDA_CHECK(h->first.reserve((size_t)batch + 1));
  B2S_CUDA_CHECK(h->range_off.reserve(batch));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->d_n_beams, n_beams, sizeof(int32_t) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->d_angle_min, angle_min, sizeof(float) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->d_angle_increment, angle_increment, sizeof(float) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->d_store_off, h->store_off.data(), sizeof(long long) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemsetAsync(h->seen, 0, sizeof(int32_t) * batch, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  *out = h.release();
  return B2S_OK;
}

extern "C" void b2s_plicp_scan_match_destroy(b2s_plicp_scan_match *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->st);
  delete h;
}

extern "C" b2s_status b2s_plicp_scan_match_reset(b2s_plicp_scan_match *h, int recording) {
  if (!h || recording < -1 || recording >= h->batch)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_reset: invalid argument");
  B2S_CUDA_CHECK(cudaSetDevice(h->device));
  const int lo = recording < 0 ? 0 : recording, cnt = recording < 0 ? h->batch : 1;
  B2S_CUDA_CHECK(cudaMemsetAsync(h->seen.p + lo, 0, sizeof(int32_t) * cnt, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  return B2S_OK;
}

extern "C" b2s_status b2s_plicp_scan_match_process(b2s_plicp_scan_match *h, const int32_t *n_scans,
                                                   const float *ranges, const float *range_limits,
                                                   b2s_plicp_scan_match_step *out) {
  B2S_NVTX("K3 PL-ICP scan match process");
  if (!h || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_process: null argument");
  const int B = h->batch;
  std::vector<long long> first(B + 1), range_off(B);
  long long total = 0, total_ranges = 0;
  int max_n = 0;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_process: negative scan count");
    first[b] = total;
    range_off[b] = total_ranges;
    total += n_scans[b];
    total_ranges += (long long)n_scans[b] * h->n_beams[b];
    if (n_scans[b] > 0) max_n = std::max(max_n, (int)h->n_beams[b]);
  }
  first[B] = total;
  if (total == 0) return B2S_OK;
  if (!ranges || !range_limits || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_scan_match_process: null array");
  if (total > 0x7fffffffLL) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_plicp_scan_match_process: more than 2^31 - 1 scans in one call");
  B2S_CUDA_CHECK(cudaSetDevice(h->device));
  B2S_CUDA_CHECK(h->ranges.reserve((size_t)total_ranges));
  B2S_CUDA_CHECK(h->limits.reserve(2 * (size_t)total));
  B2S_CUDA_CHECK(h->out.reserve((size_t)total));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->ranges, ranges, sizeof(float) * total_ranges, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->limits, range_limits, sizeof(float) * 2 * total, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->first, first.data(), sizeof(long long) * (B + 1), cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->range_off, range_off.data(), sizeof(long long) * B, cudaMemcpyHostToDevice, h->st));
  ScanMatchLaunch A;
  A.P = h->params;
  A.batch = B;
  A.n_beams = h->d_n_beams; A.angle_min = h->d_angle_min; A.angle_increment = h->d_angle_increment;
  A.first = h->first; A.range_off = h->range_off; A.store_off = h->d_store_off;
  A.ranges = h->ranges; A.limits = h->limits;
  A.store_ranges = h->store_ranges; A.store_limits = h->store_limits; A.seen = h->seen;
  A.out = h->out;
  k_plicp_scan_match<<<(unsigned)total, ICP_THREADS, scan_match_smem(max_n), h->st>>>(A);
  B2S_CUDA_CHECK(cudaGetLastError());
  k_plicp_scan_match_store<<<B, 256, 0, h->st>>>(A, h->store_ranges, h->store_limits, h->seen);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, h->out, sizeof(b2s_plicp_scan_match_step) * total, cudaMemcpyDeviceToHost, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  return B2S_OK;
}
