// K3 (lesson3) — the PL-ICP odometry node on H100 (sm_90a): ScanMatchPLICP::ScanCallback
// (reference/lesson3/src/plicp_odometry.cc:191-517) for B independent recordings of one laser, one CTA per recording,
// every scan of a call in ONE launch.
//
// Per scan the CTA converts the LaserScan into the current-scan slot of the pair kernel's shared memory, thread 0 runs
// the node's tf2 chain in double (constant-velocity prediction moved into the laser frame, :352-370), the CTA runs the
// pair matcher (plicp_pair.cuh, the code of b2s_plicp_match) against the key frame in the other slot, and thread 0
// composes the correction into base_in_odom_ (:397-413), writes the published odometry (:472-492) and decides the key
// frame (:498-517).  Promoting a scan swaps the two slots' pointers; nothing is copied in shared memory.
//
// tf2 LinearMath and ros::Duration are ros_math.cuh's, in double with no FMA contraction (-fmad=false); only the
// device's sin / cos / atan2 / sqrt may differ from glibc's in the last place.  The state between calls lives in device memory
// (PlicpOdomState, the key frame's float32 ranges), so calls over consecutive parts of a recording equal one call.
#include <cmath>
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
  int32_t reserved;
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
  b2s_plicp_odom_params P;
  int n;
  float angle_min, angle_increment, range_min, range_max;
  const int32_t *n_scans;     // [B]
  const long long *first;     // [B]: index of the recording's first scan of this call in ranges / stamps / out
  const float *ranges;        // [sum][n]
  const uint32_t *stamps;     // [sum][2]
  float *keyframe_ranges;     // [B][n]: the key frame scan of every recording (persistent)
  PlicpOdomState *state;      // [B] (persistent)
  b2s_plicp_odom_step *out;   // [sum]
};

__global__ void __launch_bounds__(ICP_THREADS) k_plicp_odometry(OdomLaunch A) {
  extern __shared__ __align__(16) unsigned char icp_smem[];
  __shared__ double red[ICP_THREADS][17];
  __shared__ double xs[8];
  __shared__ int s_cnt[4];
  __shared__ int s_promote;
  const int b = blockIdx.x, tid = threadIdx.x, n = A.n;
  const int cnt = A.n_scans[b];
  if (cnt == 0) return;
  double *kx, *ky, *cx, *cy;  // key frame slot, current scan slot
  uint8_t *kv, *cv;
  IcpPairSmem S;
  icp_carve(icp_smem, n, kx, ky, cx, cy, kv, cv, S);
  S.red = red; S.xs = xs; S.s_cnt = s_cnt;
  const double rmin = A.range_min, rmax = A.range_max;  // float32 message fields widened (:295)
  const double min_theta = beam_theta(A.angle_min, A.angle_increment, 0);
  const double max_theta = beam_theta(A.angle_min, A.angle_increment, n - 1);
  float *kf_store = A.keyframe_ranges + (size_t)b * n;
  int seen = A.state[b].scans_seen;  // every thread tracks it; only thread 0 touches the rest of the state
  PlicpOdomState st;
  TfTransform base_to_laser, laser_to_base;
  if (tid == 0) {
    st = A.state[b];
    // GetBaseToLaserTf (:257-280): tf2::fromMsg(transform, base_to_laser_), laser_to_base_ = its inverse
    const double *m = A.P.base_to_laser;
    base_to_laser.o[0] = m[0]; base_to_laser.o[1] = m[1]; base_to_laser.o[2] = m[2];
    tf_set_rotation(base_to_laser, m + 3);
    laser_to_base = tf_inverse(base_to_laser);
  }
  if (seen > 0)
    for (int i = tid; i < n; i += ICP_THREADS)
      icp_load_point(kf_store[i], beam_theta(A.angle_min, A.angle_increment, i), rmin, rmax, kx, ky, kv, i);
  const long long first = A.first[b];
  for (int s = 0; s < cnt; s++) {
    const float *r = A.ranges + (size_t)(first + s) * n;
    const uint32_t *stamp = A.stamps + 2 * (first + s);
    b2s_plicp_odom_step *o = A.out + first + s;
    if (seen == 0) {
      // the first scan initialises the node (:196-211): it becomes the key frame, nothing is published
      for (int i = tid; i < n; i += ICP_THREADS) {
        icp_load_point(r[i], beam_theta(A.angle_min, A.angle_increment, i), rmin, rmax, kx, ky, kv, i);
        kf_store[i] = r[i];
      }
      if (tid == 0) {
        tf_identity(st.base_in_odom);
        tf_identity(st.base_in_odom_keyframe);
        st.velocity_linear_x = st.velocity_angular_z = 0.0;
        st.scan_count = 0;
        st.keyframe_scan = 0;
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
      icp_load_point(r[i], beam_theta(A.angle_min, A.angle_increment, i), rmin, rmax, cx, cy, cv, i);
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
    icp_pair(A.P.icp, n, min_theta, max_theta, S, guess, &res);
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
      if (fabs(tf_yaw_of(corr)) > A.P.kf_dist_angular) {
        kf = true;
      } else if (st.scan_count == A.P.kf_scan_count) {
        st.scan_count = 0;
        kf = true;
      } else {
        const double x = corr.o[0], y = corr.o[1];
        kf = x * x + y * y > A.P.kf_dist_linear * A.P.kf_dist_linear;
      }
      if (kf) {
        st.base_in_odom_keyframe = st.base_in_odom;
        st.keyframe_scan = seen;
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
  int device = 0, batch = 0, n = 0;
  b2s_plicp_odom_params params;
  float angle_min = 0, angle_increment = 0, range_min = 0, range_max = 0;
  size_t smem = 0;
  Buf<PlicpOdomState> state;
  Buf<float> keyframe_ranges, ranges;
  Buf<uint32_t> stamps;
  Buf<int32_t> counts;
  Buf<long long> first;
  Buf<b2s_plicp_odom_step> out;
};

extern "C" b2s_status b2s_plicp_odom_create(const b2s_plicp_odom_params *params, int batch, int n_beams,
                                           float angle_min, float angle_increment, float range_min, float range_max,
                                           int device, void *cuda_stream, b2s_plicp_odom **out) {
  B2S_NVTX("K3 PL-ICP odometry create");
  if (!params || !out || batch <= 0 || n_beams < 3 || params->icp.max_iterations < 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_create: null/invalid argument");
  const double *q = params->base_to_laser + 3;
  const double q2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (!(q2 > 0.0) || !std::isfinite(q2)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_create: base_to_laser rotation is not a quaternion");
  *out = nullptr;
  if (b2s_status s = open_device(device)) return s;
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_plicp_odometry));
  int optin = 0;
  B2S_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  const size_t smem = (size_t)n_beams * ICP_SMEM_PER_BEAM + 64;
  if (smem + fa.sharedSizeBytes > (size_t)optin)
    B2S_FAIL(B2S_ERR_TOO_LARGE, "too many beams for the shared-memory PL-ICP kernel");
  B2S_CUDA_CHECK(raise_dyn_smem(k_plicp_odometry, smem));
  std::unique_ptr<b2s_plicp_odom> h(new b2s_plicp_odom());
  B2S_CUDA_CHECK(h->st.init(cuda_stream));
  h->device = device; h->batch = batch; h->n = n_beams; h->params = *params;
  h->angle_min = angle_min; h->angle_increment = angle_increment; h->range_min = range_min; h->range_max = range_max;
  h->smem = smem;
  B2S_CUDA_CHECK(h->state.reserve(batch));
  B2S_CUDA_CHECK(h->keyframe_ranges.reserve((size_t)batch * n_beams));
  B2S_CUDA_CHECK(h->counts.reserve(batch));
  B2S_CUDA_CHECK(h->first.reserve(batch));
  B2S_CUDA_CHECK(cudaMemsetAsync(h->state, 0, sizeof(PlicpOdomState) * batch, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  *out = h.release();
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

extern "C" b2s_status b2s_plicp_odom_process(b2s_plicp_odom *h, const int32_t *n_scans, const float *ranges,
                                            const uint32_t *stamps, b2s_plicp_odom_step *out) {
  B2S_NVTX("K3 PL-ICP odometry process");
  if (!h || !n_scans) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process: null argument");
  std::vector<long long> first(h->batch);
  long long total = 0;
  for (int b = 0; b < h->batch; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process: negative scan count");
    first[b] = total;
    total += n_scans[b];
  }
  if (total == 0) return B2S_OK;
  if (!ranges || !stamps || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_plicp_odom_process: null array");
  B2S_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t n = h->n;
  B2S_CUDA_CHECK(h->ranges.reserve((size_t)total * n));
  B2S_CUDA_CHECK(h->stamps.reserve(2 * (size_t)total));
  B2S_CUDA_CHECK(h->out.reserve((size_t)total));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->ranges, ranges, sizeof(float) * total * n, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->stamps, stamps, sizeof(uint32_t) * 2 * total, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->counts, n_scans, sizeof(int32_t) * h->batch, cudaMemcpyHostToDevice, h->st));
  B2S_CUDA_CHECK(cudaMemcpyAsync(h->first, first.data(), sizeof(long long) * h->batch, cudaMemcpyHostToDevice, h->st));
  OdomLaunch A;
  A.P = h->params;
  A.n = h->n;
  A.angle_min = h->angle_min; A.angle_increment = h->angle_increment;
  A.range_min = h->range_min; A.range_max = h->range_max;
  A.n_scans = h->counts; A.first = h->first; A.ranges = h->ranges; A.stamps = h->stamps;
  A.keyframe_ranges = h->keyframe_ranges; A.state = h->state; A.out = h->out;
  k_plicp_odometry<<<h->batch, ICP_THREADS, h->smem, h->st>>>(A);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, h->out, sizeof(b2s_plicp_odom_step) * total, cudaMemcpyDeviceToHost, h->st));
  B2S_CUDA_CHECK(cudaStreamSynchronize(h->st));
  return B2S_OK;
}
