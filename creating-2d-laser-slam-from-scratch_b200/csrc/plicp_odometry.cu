// K3 (lesson3) — the PL-ICP odometry node on H100 (sm_90a): ScanMatchPLICP::ScanCallback
// (reference/lesson3/src/plicp_odometry.cc:191-517) for B independent recordings, each of its own laser, mount and
// parameters, one CTA per recording, every scan of a call in ONE launch.
//
// Per scan the CTA converts the LaserScan into the current-scan slot of the pair kernel's shared memory (LaserScanToLDP,
// :285-322, with the message's own range fields), thread 0 runs the node's tf2 chain in double (constant-velocity
// prediction moved into the laser frame, :352-370), the CTA runs the pair matcher (plicp_pair.cuh, the code of
// b2s_plicp_match) against the key frame in the other slot, and thread 0 composes the correction into base_in_odom_
// (:397-413), writes the published odometry (:472-492) and decides the key frame (:498-517).  Promoting a scan swaps the
// two slots' pointers; nothing is copied in shared memory.
//
// tf2 LinearMath and ros::Duration are ros_math.cuh's, in double with no FMA contraction (-fmad=false); only the
// device's sin / cos / atan2 / sqrt may differ from glibc's in the last place.  The state between calls lives in device
// memory (PlicpOdomState, the key frame's float32 ranges and the range fields it was converted with), so calls over
// consecutive parts of a recording equal one call.
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"
#include "plicp_pair.cuh"
#include "ros_math.cuh"

using namespace b2s;

namespace b2s {

// per-recording state of the node between scans
struct PlicpOdomState {
  TfTransform base_in_odom, base_in_odom_keyframe;
  double velocity_linear_x, velocity_angular_z;  // latest_velocity_ (the node sets no other field)
  uint32_t last_sec, last_nsec;                   // last_icp_time_
  int32_t scan_count;                             // scan_count_
  int32_t keyframe_scan;                          // index in the recording of the key frame scan
  int32_t scans_seen;                             // scans of the recording processed so far (0: not initialised)
  float kf_range_min, kf_range_max;               // the key frame message's range fields (prev_ldp_scan_'s valid flags)
};

__device__ inline double tf_yaw_of(const TfTransform &t) {
  double q[4];
  tf_get_rotation(t, q);
  return tf2_get_yaw(q);
}

// ScanMatchPLICP::CreateTfFromXYTheta (:461-467): origin (x, y, 0), rotation Quaternion::setRPY(0, 0, theta)
__device__ inline TfTransform tf_from_xyt(double x, double y, double theta) {
  double q[4];
  quat_set_rpy(0.0, 0.0, theta, q);
  TfTransform t;
  t.o[0] = x; t.o[1] = y; t.o[2] = 0.0;
  tf_set_rotation(t, q);
  return t;
}

// LaserScanToLDP's beam angle (:308): angle_min + i * angle_increment summed in float, then widened
__device__ __forceinline__ double beam_theta(float angle_min, float angle_increment, int i) {
  return (double)__fadd_rn(angle_min, __fmul_rn((float)i, angle_increment));
}

struct OdomLaunch {
  const b2s_plicp_odom_params *__restrict__ params;  // [B]
  const b2s_plicp_odom_laser *lasers;   // [B]
  const long long *first;               // [B + 1]: index of recording b's first scan of this call in limits / stamps / out
  const long long *range_off;           // [B]: offset of recording b's first scan of this call in ranges
  const long long *store_off;           // [B]: offset of recording b's key frame in keyframe_ranges
  const float *ranges;                  // [sum over b of n_scans[b] * n_beams[b]]
  const float *limits;                  // [sum][2]: range_min, range_max of every scan
  const uint32_t *stamps;               // [sum][2]
  float *keyframe_ranges;               // [sum n_beams]: the key frame scan of every recording (persistent)
  PlicpOdomState *state;                // [B] (persistent)
  b2s_plicp_odom_step *out;             // [sum]
};

__global__ void __launch_bounds__(ICP_THREADS) k_plicp_odometry(OdomLaunch A) {
  extern __shared__ __align__(16) unsigned char icp_smem[];
  __shared__ double red[ICP_THREADS][17];
  __shared__ double xs[8];
  __shared__ int s_cnt[4];
  __shared__ int s_promote;
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long first = A.first[b];
  const int cnt = (int)(A.first[b + 1] - first);
  if (cnt == 0) return;
  // the recording's parameters stay in global memory (read through L1): at the pair kernel's beam limit its shared
  // memory leaves 16 bytes free, too few for the 176-byte row
  const b2s_plicp_odom_params &P = A.params[b];
  const b2s_plicp_odom_laser laser = A.lasers[b];
  const int n = laser.n_beams;
  double *kx, *ky, *cx, *cy;  // key frame slot, current scan slot
  uint8_t *kv, *cv;
  IcpPairSmem S;
  icp_carve(icp_smem, n, kx, ky, cx, cy, kv, cv, S);
  S.red = red; S.xs = xs; S.s_cnt = s_cnt;
  const double min_theta = beam_theta(laser.angle_min, laser.angle_increment, 0);
  const double max_theta = beam_theta(laser.angle_min, laser.angle_increment, n - 1);
  float *kf_store = A.keyframe_ranges + A.store_off[b];
  int seen = A.state[b].scans_seen;  // every thread tracks it; only thread 0 touches the rest of the state
  PlicpOdomState st;
  TfTransform base_to_laser, laser_to_base;
  if (tid == 0) {
    st = A.state[b];
    // GetBaseToLaserTf (:257-280): tf2::fromMsg(transform, base_to_laser_), laser_to_base_ = its inverse
    const double *m = P.base_to_laser;
    base_to_laser.o[0] = m[0]; base_to_laser.o[1] = m[1]; base_to_laser.o[2] = m[2];
    tf_set_rotation(base_to_laser, m + 3);
    laser_to_base = tf_inverse(base_to_laser);
  }
  if (seen > 0) {
    // the key frame as its own message's fields converted it (float32 fields widened, :295)
    const double kmin = A.state[b].kf_range_min, kmax = A.state[b].kf_range_max;
    for (int i = tid; i < n; i += ICP_THREADS)
      icp_load_point(kf_store[i], beam_theta(laser.angle_min, laser.angle_increment, i), kmin, kmax, kx, ky, kv, i);
  }
  for (int s = 0; s < cnt; s++) {
    const float *r = A.ranges + A.range_off[b] + (size_t)s * n;
    const float *lim = A.limits + 2 * (first + s);
    const uint32_t *stamp = A.stamps + 2 * (first + s);
    b2s_plicp_odom_step *o = A.out + first + s;
    const double rmin = lim[0], rmax = lim[1];  // this message's float32 fields widened (:295)
    if (seen == 0) {
      // the first scan initialises the node (:196-211): it becomes the key frame, nothing is published
      for (int i = tid; i < n; i += ICP_THREADS) {
        icp_load_point(r[i], beam_theta(laser.angle_min, laser.angle_increment, i), rmin, rmax, kx, ky, kv, i);
        kf_store[i] = r[i];
      }
      if (tid == 0) {
        tf_identity(st.base_in_odom);
        tf_identity(st.base_in_odom_keyframe);
        st.velocity_linear_x = st.velocity_angular_z = 0.0;
        st.scan_count = 0;
        st.keyframe_scan = 0;
        st.kf_range_min = lim[0]; st.kf_range_max = lim[1];
        st.last_sec = stamp[0]; st.last_nsec = stamp[1];
        b2s_plicp_odom_step z = {};
        z.orientation[3] = 1.0;
        z.keyframe = 1;
        z.reference_scan = -1;
        *o = z;
      }
      seen = 1;
      __syncthreads();
      continue;
    }
    for (int i = tid; i < n; i += ICP_THREADS)
      icp_load_point(r[i], beam_theta(laser.angle_min, laser.angle_increment, i), rmin, rmax, cx, cy, cv, i);
    double guess[3] = {0.0, 0.0, 0.0}, dt = 0.0;
    if (tid == 0) {
      // dt = (time - last_icp_time_).toSec()
      dt = ros_duration_to_sec(ros_time_diff(stamp[0], stamp[1], st.last_sec, st.last_nsec));
      // GetPrediction (:442-456): only linear.x is ever set; linear.y and linear.z (the angle) are 0
      const double pr_x = st.velocity_linear_x < 1e-6 ? 0.0 : dt * st.velocity_linear_x;
      const double pr_y = 0.0, pr_a = 0.0;
      TfTransform pc = tf_from_xyt(pr_x, pr_y, pr_a);
      pc = tf_mul(pc, tf_mul(st.base_in_odom, tf_inverse(st.base_in_odom_keyframe)));
      const TfTransform pcl = tf_mul(tf_mul(tf_mul(tf_mul(laser_to_base, tf_inverse(st.base_in_odom)), pc), st.base_in_odom),
                            base_to_laser);
      guess[0] = pcl.o[0];
      guess[1] = pcl.o[1];
      guess[2] = tf_yaw_of(pcl);
    }
    b2s_icp_result res;
    S.rx = kx; S.ry = ky; S.rv = kv; S.sx = cx; S.sy = cy; S.sv = cv;
    icp_pair(P.icp, n, min_theta, max_theta, S, guess, &res);
    if (tid == 0) {
      TfTransform corr;
      tf_identity(corr);  // a failed match leaves corr_ch default-constructed: taken as the identity (DESIGN.md §7)
      if (res.valid) {
        const TfTransform corr_l = tf_from_xyt(res.x[0], res.x[1], res.x[2]);
        corr = tf_mul(tf_mul(base_to_laser, corr_l), laser_to_base);
        st.base_in_odom = tf_mul(st.base_in_odom_keyframe, corr);
        st.velocity_linear_x = corr.o[0] / dt;
        st.velocity_angular_z = tf_yaw_of(corr) / dt;
      }
      // PublishTFAndOdometry (:472-492)
      b2s_plicp_odom_step z = {};
      for (int q = 0; q < 3; q++) z.position[q] = st.base_in_odom.o[q];
      tf_get_rotation(st.base_in_odom, z.orientation);
      z.linear[0] = st.velocity_linear_x;
      z.angular[2] = st.velocity_angular_z;
      for (int q = 0; q < 3; q++) z.first_guess[q] = guess[q];
      z.icp = res;
      z.published = 1;
      z.reference_scan = st.keyframe_scan;
      // NewKeyframeNeeded (:498-517)
      bool kf;
      st.scan_count++;
      if (fabs(tf_yaw_of(corr)) > P.kf_dist_angular) {
        kf = true;
      } else if (st.scan_count == P.kf_scan_count) {
        st.scan_count = 0;
        kf = true;
      } else {
        const double x = corr.o[0], y = corr.o[1];
        kf = x * x + y * y > P.kf_dist_linear * P.kf_dist_linear;
      }
      if (kf) {
        st.base_in_odom_keyframe = st.base_in_odom;
        st.keyframe_scan = seen;
        st.kf_range_min = lim[0]; st.kf_range_max = lim[1];
      }
      z.keyframe = kf;
      *o = z;
      st.last_sec = stamp[0]; st.last_nsec = stamp[1];
      s_promote = kf;
    }
    seen++;
    __syncthreads();
    if (s_promote) {
      for (int i = tid; i < n; i += ICP_THREADS) kf_store[i] = r[i];
      double *t;
      t = kx; kx = cx; cx = t;
      t = ky; ky = cy; cy = t;
      uint8_t *v = kv; kv = cv; cv = v;
    }
    __syncthreads();
  }
  if (tid == 0) {
    st.scans_seen = seen;
    A.state[b] = st;
  }
}

}  // namespace b2s

struct b2s_plicp_odom {
  Stream st;  // declared first: destroyed after the buffers
  int device = 0, batch = 0;
  bool has_fields = false;               // made by b2s_plicp_odom_create: range_min / range_max fixed for every scan
  float range_min = 0, range_max = 0;
  std::vector<int32_t> n_beams;
  Buf<b2s_plicp_odom_params> params;
  Buf<b2s_plicp_odom_laser> lasers;
  Buf<PlicpOdomState> state;
  Buf<float> keyframe_ranges, ranges, limits;
  Buf<uint32_t> stamps;
  Buf<long long> store_off, offsets;     // offsets: first [B + 1], then range_off [B] of the current call
  Buf<b2s_plicp_odom_step> out;
};

// the pair kernel's dynamic shared memory for n beams
static size_t odom_smem(int n) { return (size_t)n * ICP_SMEM_PER_BEAM + 64; }

// The fleet behind both create entry points: recording b's parameters are params[b * stride] and its laser
// lasers[b * stride] (stride 0: one row for all).  `api` names the entry point in refusals, with the recording when
// the rows differ.
static b2s_status odom_create(int batch, const b2s_plicp_odom_params *params, const b2s_plicp_odom_laser *lasers,
                              int stride, int device, void *cuda_stream, b2s_plicp_odom **out, const char *api) {
  if (!out) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": null argument");
  *out = nullptr;
  if (!params || !lasers) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": null argument");
  if (batch < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(api) + ": batch must be positive");
  auto who = [&](int b) {
    return stride ? std::string(api) + ": recording " + std::to_string(b) + ": " : std::string(api) + ": ";
  };
  int max_n = 0;
  for (int b = 0; b < batch; b++) {
    const b2s_plicp_odom_params &p = params[(size_t)b * stride];
    const b2s_plicp_odom_laser &l = lasers[(size_t)b * stride];
    if (l.n_beams < 3) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "fewer than 3 beams");
    if (l.reserved != 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "laser reserved field is not 0");
    if (p.icp.max_iterations < 1) B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "icp.max_iterations must be positive");
    const double *q = p.base_to_laser + 3;
    const double q2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    if (!(q2 > 0.0) || !std::isfinite(q2))
      B2S_FAIL(B2S_ERR_BAD_PARAMS, who(b) + "base_to_laser rotation is not a quaternion");
    max_n = std::max(max_n, (int)l.n_beams);
  }
  if (b2s_status s = open_device(device)) return s;
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_plicp_odometry));
  int optin = 0;
  B2S_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  for (int b = 0; b < batch; b++)
    if (odom_smem(lasers[(size_t)b * stride].n_beams) + fa.sharedSizeBytes > (size_t)optin)
      B2S_FAIL(B2S_ERR_TOO_LARGE, who(b) + "too many beams for the shared-memory PL-ICP kernel");
  B2S_CUDA_CHECK(raise_dyn_smem(k_plicp_odometry, odom_smem(max_n)));
  std::unique_ptr<b2s_plicp_odom> h(new b2s_plicp_odom());
  B2S_CUDA_CHECK(h->st.init(cuda_stream));
  h->device = device; h->batch = batch;
  std::vector<b2s_plicp_odom_params> P((size_t)batch);
  std::vector<b2s_plicp_odom_laser> Ls((size_t)batch);
  std::vector<long long> store_off((size_t)batch);
  h->n_beams.resize((size_t)batch);
  long long total_beams = 0;
  for (int b = 0; b < batch; b++) {
    P[(size_t)b] = params[(size_t)b * stride];
    Ls[(size_t)b] = lasers[(size_t)b * stride];
    h->n_beams[(size_t)b] = Ls[(size_t)b].n_beams;
    store_off[(size_t)b] = total_beams;
    total_beams += Ls[(size_t)b].n_beams;
  }
  B2S_CUDA_CHECK(h->params.reserve(batch));
  B2S_CUDA_CHECK(h->lasers.reserve(batch));
  B2S_CUDA_CHECK(h->state.reserve(batch));
  B2S_CUDA_CHECK(h->keyframe_ranges.reserve((size_t)total_beams));
  B2S_CUDA_CHECK(h->store_off.reserve(batch));
  B2S_CUDA_CHECK(h->offsets.reserve(2 * (size_t)batch + 1));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->params, P.data(), sizeof(b2s_plicp_odom_params) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->lasers, Ls.data(), sizeof(b2s_plicp_odom_laser) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->store_off, store_off.data(), sizeof(long long) * batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemsetAsync(h->state, 0, sizeof(PlicpOdomState) * batch, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  *out = h.release();
  return B2S_OK;
}

extern "C" b2s_status b2s_plicp_odom_create_fleet(int batch, const b2s_plicp_odom_params *params,
                                                 const b2s_plicp_odom_laser *lasers, int device, void *cuda_stream,
                                                 b2s_plicp_odom **out) {
  B2S_NVTX("K3 PL-ICP odometry create");
  return odom_create(batch, params, lasers, 1, device, cuda_stream, out, "b2s_plicp_odom_create_fleet");
}

extern "C" b2s_status b2s_plicp_odom_create(const b2s_plicp_odom_params *params, int batch, int n_beams,
                                           float angle_min, float angle_increment, float range_min, float range_max,
                                           int device, void *cuda_stream, b2s_plicp_odom **out) {
  B2S_NVTX("K3 PL-ICP odometry create");
  const b2s_plicp_odom_laser laser = {n_beams, angle_min, angle_increment, 0};
  if (b2s_status s = odom_create(batch, params, &laser, 0, device, cuda_stream, out, "b2s_plicp_odom_create")) return s;
  (*out)->has_fields = true;
  (*out)->range_min = range_min;
  (*out)->range_max = range_max;
  return B2S_OK;
}

extern "C" void b2s_plicp_odom_destroy(b2s_plicp_odom *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->st);
  delete h;
}

extern "C" b2s_status b2s_plicp_odom_reset(b2s_plicp_odom *h, int recording) {
  if (!h || recording < -1 || recording >= h->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_reset: invalid argument");
  B2S_CUDA_CHECK(cudaSetDevice(h->device));
  const int lo = recording < 0 ? 0 : recording, cnt = recording < 0 ? h->batch : 1;
  B2S_CUDA_CHECK(cudaMemsetAsync(h->state.p + lo, 0, sizeof(PlicpOdomState) * cnt, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  return B2S_OK;
}

extern "C" b2s_status b2s_plicp_odom_process_fleet(b2s_plicp_odom *h, const int32_t *n_scans, const float *ranges,
                                                  const float *range_limits, const uint32_t *stamps,
                                                  b2s_plicp_odom_step *out) {
  B2S_NVTX("K3 PL-ICP odometry process");
  if (!h || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process_fleet: null argument");
  const int B = h->batch;
  std::vector<long long> offs(2 * (size_t)B + 1);  // first [B + 1], range_off [B]
  long long total = 0, total_ranges = 0;
  int max_n = 0;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process_fleet: negative scan count");
    offs[(size_t)b] = total;
    offs[(size_t)B + 1 + b] = total_ranges;
    total += n_scans[b];
    total_ranges += (long long)n_scans[b] * h->n_beams[(size_t)b];
    if (n_scans[b] > 0) max_n = std::max(max_n, (int)h->n_beams[(size_t)b]);
  }
  offs[(size_t)B] = total;
  if (total == 0) return B2S_OK;
  if (total > 0x7fffffffLL) B2S_FAIL(B2S_ERR_TOO_LARGE, "b2s_plicp_odom_process_fleet: more than 2^31 - 1 scans in one call");
  if (!ranges || !range_limits || !stamps || !out)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process_fleet: null array");
  B2S_CUDA_CHECK(cudaSetDevice(h->device));
  B2S_CUDA_CHECK(h->ranges.reserve((size_t)total_ranges));
  B2S_CUDA_CHECK(h->limits.reserve(2 * (size_t)total));
  B2S_CUDA_CHECK(h->stamps.reserve(2 * (size_t)total));
  B2S_CUDA_CHECK(h->out.reserve((size_t)total));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->ranges, ranges, sizeof(float) * total_ranges, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->limits, range_limits, sizeof(float) * 2 * total, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->stamps, stamps, sizeof(uint32_t) * 2 * total, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->offsets, offs.data(), sizeof(long long) * offs.size(), cudaMemcpyHostToDevice, h->st));
  OdomLaunch A;
  A.params = h->params; A.lasers = h->lasers;
  A.first = h->offsets; A.range_off = h->offsets.p + B + 1; A.store_off = h->store_off;
  A.ranges = h->ranges; A.limits = h->limits; A.stamps = h->stamps;
  A.keyframe_ranges = h->keyframe_ranges; A.state = h->state; A.out = h->out;
  k_plicp_odometry<<<B, ICP_THREADS, odom_smem(max_n), h->st>>>(A);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, h->out, sizeof(b2s_plicp_odom_step) * total, cudaMemcpyDeviceToHost, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  return B2S_OK;
}

extern "C" b2s_status b2s_plicp_odom_process(b2s_plicp_odom *h, const int32_t *n_scans, const float *ranges,
                                            const uint32_t *stamps, b2s_plicp_odom_step *out) {
  if (!h || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process: null argument");
  if (!h->has_fields)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process: a fleet handle has no create-time range fields (use "
                                 "b2s_plicp_odom_process_fleet)");
  long long total = 0;
  for (int b = 0; b < h->batch; b++) total += n_scans[b] > 0 ? n_scans[b] : 0;
  std::vector<float> limits;
  if (total <= 0x7fffffffLL) {  // larger calls are refused by process_fleet before it reads the limits
    limits.resize(2 * (size_t)total);
    for (long long s = 0; s < total; s++) {
      limits[(size_t)(2 * s)] = h->range_min;
      limits[(size_t)(2 * s + 1)] = h->range_max;
    }
  }
  return b2s_plicp_odom_process_fleet(h, n_scans, ranges, limits.empty() ? nullptr : limits.data(), stamps, out);
}
