// TEST HELPER: the nvcc DEVICE build of the library's shared math headers (glibc_math.cuh, ros_math.cuh, common.cuh,
// hector_grid.cuh) against their host build and the C library, function by function.  Built with the library's own
// nvcc flags (build.NVCC_FLAGS) and -Xcompiler -ffp-contract=off, linked against libm; tests/test_gpu_device_math.py
// runs it on the GPU, tests/test_device_math_host.py runs its host half only.
//
// usage: device_math_check [--host-only] [--out DIR]
// Prints one JSON line per group: "group", "inputs", "mismatches", "first" (up to 20 mismatching inputs as hex bits,
// smallest first) and group-specific counts.  The groups evaluated against mpmath (ros_math_libm, and sensor_pose_of in
// common_helpers) also write their records to DIR/libm_records.bin: float64 rows of
// [op, in[0..8], device out[0..3], host out[0..3]] (device columns NaN with --host-only).
//
// Exhaustive groups run in chunks of 2^26 inputs on one stream: kernel, copy back, compare on all host threads.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../creating-2d-laser-slam-from-scratch_b200/csrc/common.cuh"
#include "../creating-2d-laser-slam-from-scratch_b200/csrc/glibc_math.cuh"
#include "../creating-2d-laser-slam-from-scratch_b200/csrc/hector_grid.cuh"
#include "../creating-2d-laser-slam-from-scratch_b200/csrc/ros_math.cuh"
#include "ros_math_sweep.h"

using namespace b2s;

namespace {

#define CK(expr)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (expr);                                                                  \
    if (e_ != cudaSuccess) {                                                                  \
      std::fprintf(stderr, "%s failed: %s (line %d)\n", #expr, cudaGetErrorString(e_), __LINE__); \
      std::exit(2);                                                                           \
    }                                                                                         \
  } while (0)

constexpr size_t CHUNK = size_t(1) << 26;
constexpr uint32_t SIGN = 0x80000000u;

uint32_t fbits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
float bfloat(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
uint64_t dbits(double d) { uint64_t u; std::memcpy(&u, &d, 8); return u; }
bool same_f(float a, float b) { return (std::isnan(a) && std::isnan(b)) || fbits(a) == fbits(b); }
bool same_d(double a, double b) { return (std::isnan(a) && std::isnan(b)) || dbits(a) == dbits(b); }

int n_threads() { return (int)std::max(1u, std::thread::hardware_concurrency()); }

// f(begin, end) over [0, n) split across the host threads
template <class F>
void parallel_for(size_t n, F f) {
  const int nt = n_threads();
  std::vector<std::thread> th;
  const size_t per = (n + nt - 1) / nt;
  for (int t = 0; t < nt; t++) {
    const size_t b = std::min(n, per * t), e = std::min(n, per * (t + 1));
    if (b < e) th.emplace_back(f, b, e);
  }
  for (auto &x : th) x.join();
}

// mismatch counter of one group: the count and the smallest mismatching inputs
struct Misses {
  std::atomic<long> n{0};
  std::mutex mu;
  std::vector<std::string> first;
  void add(const std::string &what) {
    n++;
    std::lock_guard<std::mutex> lock(mu);
    first.push_back(what);
    std::sort(first.begin(), first.end());
    if (first.size() > 20) first.resize(20);
  }
  std::string json() {
    std::string s = "[";
    for (size_t i = 0; i < first.size(); i++) s += (i ? ", \"" : "\"") + first[i] + "\"";
    return s + "]";
  }
};
std::string hex32(uint32_t u) { char b[16]; std::snprintf(b, sizeof b, "0x%08x", u); return b; }
std::string hex64(double d) { char b[24]; std::snprintf(b, sizeof b, "0x%016llx", (unsigned long long)dbits(d)); return b; }

// ---------------------------------------------------------------- glibc_sincosf, both builds

__global__ void k_sincosf(const uint32_t *__restrict__ in, size_t n, bool use_fma, float4 *__restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float y = __uint_as_float(in[i]);
  float s, c;
  glibc_sincosf(y, use_fma, &s, &c);
  out[i] = make_float4(glibc_sinf(y, use_fma), glibc_cosf(y, use_fma), s, c);
}

void host_sincosf(float y, bool use_fma, float r[4]) {
  r[0] = glibc_sinf(y, use_fma);
  r[1] = glibc_cosf(y, use_fma);
  glibc_sincosf(y, use_fma, &r[2], &r[3]);
}
// the C library: sinf, cosf, sincosf
void libm_sincosf(float y, float r[4]) {
  volatile float vy = y;
  r[0] = sinf(vy);
  r[1] = cosf(vy);
  sincosf(vy, &r[2], &r[3]);
}
bool below_120(uint32_t u) { return (u & 0x7fffffffu) < 0x42f00000u; }

// every float with |x| < 120 at stride 61, both signs
std::vector<uint32_t> stride_sweep() {
  std::vector<uint32_t> v;
  for (uint32_t u = 0; u < 0x42f00000u; u += 61) { v.push_back(u); v.push_back(u | SIGN); }
  return v;
}

std::vector<uint32_t> sincosf_inputs() {
  std::vector<uint32_t> v = stride_sweep();
  auto both = [&](int64_t u) {
    if (u < 0 || u > 0x7fffffffLL) return;
    v.push_back((uint32_t)u);
    v.push_back((uint32_t)u | SIGN);
  };
  // every float within 2^16 ulps of each multiple of pi/2 below 120 (k = 0: zero and the subnormals above it)
  for (int k = 0; k * 1.5707963267948966 < 120.0; k++) {
    const int64_t c = fbits((float)(k * 1.5707963267948966));
    for (int64_t d = -65536; d <= 65536; d++)
      if (below_120((uint32_t)std::max<int64_t>(c + d, 0))) both(c + d);
  }
  // the probes that tell the two glibc builds apart, +-1024 ulps
  const uint32_t probes[17] = {0x418a3adbu, 0x418a3adcu, 0x418a3addu, 0x418a3adeu, 0x41bc76d9u, 0x4202eb4bu,
                               0x4255b0a9u, 0x42687a55u, 0x4280ce28u, 0x42870e40u, 0x42a35c07u, 0x42a35d44u,
                               0x42a97360u, 0x42c55faau, 0x42cf5854u, 0x42d8d23eu, 0x42e87a55u};
  for (uint32_t p : probes)
    for (int d = -1024; d <= 1024; d++) both((int64_t)p + d);
  // both sides of the `top` thresholds: 2^-12, pi/4's exponent, 120's exponent
  for (uint32_t top : {0x398u, 0x3f4u, 0x42fu})
    for (int d = -256; d < 256; d++) both((int64_t)(top << 20) + d);
  // +-0, subnormals, +-inf, NaNs, and the fallback range
  for (uint32_t u : {0u, 1u, 2u, 0x400000u, 0x7fffffu, 0x800000u, 0x7f800000u, 0x7fc00000u, 0x7f800001u, 0x7fffffffu,
                     0x42f00000u, 0x43000000u, 0x49742400u, 0x5f000000u, 0x7f7fffffu})
    both(u);
  return v;
}

void group_sincosf(bool use_fma, int host_variant) {
  const std::vector<uint32_t> in = sincosf_inputs();
  const size_t n = in.size();
  uint32_t *d_in = nullptr;
  float4 *d_out = nullptr;
  const size_t chunk = std::min(n, CHUNK);
  CK(cudaMalloc(&d_in, chunk * sizeof(uint32_t)));
  CK(cudaMalloc(&d_out, chunk * sizeof(float4)));
  std::vector<float4> out(chunk);
  Misses miss, libm_miss;
  std::atomic<long> below{0}, above{0}, above_differ{0}, nan_not_nan{0};
  const bool vs_libm = (use_fma ? 1 : 0) == host_variant;
  for (size_t base = 0; base < n; base += chunk) {
    const size_t m = std::min(chunk, n - base);
    CK(cudaMemcpy(d_in, in.data() + base, m * sizeof(uint32_t), cudaMemcpyHostToDevice));
    k_sincosf<<<(unsigned)((m + 255) / 256), 256>>>(d_in, m, use_fma, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out.data(), d_out, m * sizeof(float4), cudaMemcpyDeviceToHost));
    parallel_for(m, [&](size_t b, size_t e) {
      long nb = 0, na = 0, nad = 0, nnan = 0;
      for (size_t i = b; i < e; i++) {
        const uint32_t u = in[base + i];
        const float y = bfloat(u);
        const float dev[4] = {out[i].x, out[i].y, out[i].z, out[i].w};
        float host[4];
        host_sincosf(y, use_fma, host);
        bool differ = false;
        for (int k = 0; k < 4; k++) differ |= !same_f(dev[k], host[k]);
        if (below_120(u)) {
          nb++;
          if (differ) miss.add(hex32(u));
          if (vs_libm) {
            float ref[4];
            libm_sincosf(y, ref);
            bool dl = false;
            for (int k = 0; k < 4; k++) dl |= !same_f(dev[k], ref[k]);
            if (dl) libm_miss.add(hex32(u));
          }
        } else {
          na++;
          nad += differ;
          if (std::isnan(y))
            for (int k = 0; k < 4; k++) nnan += !std::isnan(dev[k]);
        }
      }
      below += nb; above += na; above_differ += nad; nan_not_nan += nnan;
    });
  }
  CK(cudaFree(d_in));
  CK(cudaFree(d_out));
  std::printf("{\"group\": \"glibc_sincosf_%s\", \"inputs\": %zu, \"inputs_below_120\": %ld, \"mismatches\": %ld, "
              "\"first\": %s, \"libm_compared\": %s, \"libm_mismatches\": %ld, \"libm_first\": %s, "
              "\"inputs_above_120\": %ld, \"above_120_differ\": %ld, \"nan_not_nan\": %ld}\n",
              use_fma ? "fma" : "plain", n, below.load(), miss.n.load(), miss.json().c_str(), vs_libm ? "true" : "false",
              libm_miss.n.load(), libm_miss.json().c_str(), above.load(), above_differ.load(), nan_not_nan.load());
  std::fflush(stdout);
}

// host half: the host restatement of each build against the C library on the stride sweep
void group_sincosf_host(bool use_fma) {
  const std::vector<uint32_t> in = stride_sweep();
  Misses miss;
  parallel_for(in.size(), [&](size_t b, size_t e) {
    for (size_t i = b; i < e; i++) {
      float host[4], ref[4];
      host_sincosf(bfloat(in[i]), use_fma, host);
      libm_sincosf(bfloat(in[i]), ref);
      bool d = false;
      for (int k = 0; k < 4; k++) d |= !same_f(host[k], ref[k]);
      if (d) miss.add(hex32(in[i]));
    }
  });
  std::printf("{\"group\": \"host_glibc_sincosf_%s\", \"inputs\": %zu, \"libm_mismatches\": %ld, \"first\": %s}\n",
              use_fma ? "fma" : "plain", in.size(), miss.n.load(), miss.json().c_str());
  std::fflush(stdout);
}

// ---------------------------------------------------------------- exhaustive float domains

// every float in [-neg_max, pos_max] (bit patterns 0..pos_max and SIGN | 0..neg_max), by index
struct Domain {
  uint32_t pos_max, neg_max;
  size_t size() const { return (size_t)pos_max + 1 + neg_max + 1; }
  __host__ __device__ uint32_t bits(size_t i) const {
    return i <= pos_max ? (uint32_t)i : (uint32_t)(i - pos_max - 1) | 0x80000000u;
  }
};

// Hector exact mode's sinRot / cosRot (hs_trig), and the de-skew's separate (float)cos / (float)sin of a double angle
__global__ void k_trig_exact(Domain dom, size_t base, size_t n, float2 *__restrict__ out,
                             unsigned long long *__restrict__ separate_differ) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = __uint_as_float(dom.bits(base + i));
  float s, c;
  libm_sincos_to_float(a, &s, &c);
  const float s1 = (float)sin((double)a), c1 = (float)cos((double)a);
  if (__float_as_uint(s1) != __float_as_uint(s) || __float_as_uint(c1) != __float_as_uint(c)) atomicAdd(separate_differ, 1ull);
  out[i] = make_float2(s, c);
}

// Hector exact mode's published probability (log_odds_prob), and the odds it rounds to float on the way
__global__ void k_prob_exact(Domain dom, size_t base, size_t n, float2 *__restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float lo = __uint_as_float(dom.bits(base + i));
  out[i] = make_float2((float)exp((double)lo), log_odds_prob(lo));
}

template <class Launch, class Ref>
void group_exhaustive(const char *name, Domain dom, Launch launch, Ref ref, const char *extra_key,
                      unsigned long long *d_extra) {
  const size_t n = dom.size();
  float2 *d_out = nullptr;
  CK(cudaMalloc(&d_out, CHUNK * sizeof(float2)));
  float2 *out = nullptr;
  CK(cudaMallocHost(&out, CHUNK * sizeof(float2)));
  Misses miss;
  for (size_t base = 0; base < n; base += CHUNK) {
    const size_t m = std::min(CHUNK, n - base);
    launch(base, m, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out, m * sizeof(float2), cudaMemcpyDeviceToHost));
    parallel_for(m, [&](size_t b, size_t e) {
      for (size_t i = b; i < e; i++) {
        const uint32_t u = dom.bits(base + i);
        float r0, r1;
        ref(bfloat(u), r0, r1);
        if (!same_f(out[i].x, r0) || !same_f(out[i].y, r1)) miss.add(hex32(u));
      }
    });
  }
  unsigned long long extra = 0;
  if (d_extra) CK(cudaMemcpy(&extra, d_extra, sizeof extra, cudaMemcpyDeviceToHost));
  CK(cudaFree(d_out));
  CK(cudaFreeHost(out));
  std::printf("{\"group\": \"%s\", \"inputs\": %zu, \"mismatches\": %ld, \"first\": %s", name, n, miss.n.load(),
              miss.json().c_str());
  if (extra_key) std::printf(", \"%s\": %llu", extra_key, extra);
  std::printf("}\n");
  std::fflush(stdout);
}

// ---------------------------------------------------------------- records: ros_math and common.cuh helpers

enum Op {
  // ros_math_arith: bit-identical
  OP_SET_ROTATION, OP_GET_ROTATION, OP_CHAIN_STEP, OP_TIME_DIFF, OP_FROM_SEC, OP_DURATION_GT,
  // ros_math_libm: against mpmath
  OP_SET_RPY, OP_GET_RPY, OP_TF_GET_YAW, OP_TF2_GET_YAW,
  // common_helpers: bit-identical, sensor_pose_of against mpmath
  OP_KROUND, OP_CAST_I32, OP_CAST_U32, OP_NORMALIZE_ANGLE, OP_NORMALIZE_DIFF, OP_WORLD_TO_GRID, OP_N_STEPS,
  OP_SENSOR_POSE,
  N_OPS
};
const char *const OP_NAMES[N_OPS] = {"set_rotation", "get_rotation", "chain_step", "time_diff", "from_sec",
                                     "duration_gt", "set_rpy", "get_rpy", "tf_get_yaw", "tf2_get_yaw", "kround",
                                     "cast_i32", "cast_u32", "normalize_angle", "normalize_angle_difference",
                                     "world_to_grid_1", "n_steps", "sensor_pose_of"};
const int OP_N_IN[N_OPS] = {4, 9, 23, 4, 1, 2, 3, 9, 4, 4, 1, 1, 1, 1, 2, 3, 2, 6};
bool op_is_libm(int op) { return (op >= OP_SET_RPY && op <= OP_TF2_GET_YAW) || op == OP_SENSOR_POSE; }
const char *op_group(int op) {
  return op <= OP_DURATION_GT ? "ros_math_arith" : op <= OP_TF2_GET_YAW ? "ros_math_libm" : "common_helpers";
}

constexpr int NIN = 24, NOUT = 16;
struct Rec {
  int op;
  double in[NIN];
};

__host__ __device__ void tf_load(TfTransform &t, const double *p) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) t.m[i][j] = p[3 * i + j];
    t.o[i] = p[9 + i];
  }
}
__host__ __device__ void tf_store(const TfTransform &t, double *p) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) p[3 * i + j] = t.m[i][j];
    p[9 + i] = t.o[i];
  }
}

// one record, the same source for both builds
__host__ __device__ void eval_op(const Rec &r, double *out) {
  for (int k = 0; k < NOUT; k++) out[k] = 0.0;
  const double *in = r.in;
  TfTransform t;
  switch (r.op) {
    case OP_SET_ROTATION:
      tf_identity(t);
      tf_set_rotation(t, in);
      tf_store(t, out);
      break;
    case OP_GET_ROTATION:
      tf_identity(t);
      for (int i = 0; i < 9; i++) t.m[i / 3][i % 3] = in[i];
      tf_get_rotation(t, out);
      break;
    case OP_CHAIN_STEP: {  // in: acc (12), q2 (4), o2 (3), v (3), kind; out: next (12), next(v) (3)
      TfTransform acc, b, next;
      tf_load(acc, in);
      tf_set_rotation(b, in + 12);
      for (int i = 0; i < 3; i++) b.o[i] = in[16 + i];
      const int kind = (int)in[22];
      if (kind == 0) next = tf_mul(acc, tf_inverse(b));
      else if (kind == 1) next = tf_mul(b, acc);
      else next = tf_inverse(tf_mul(acc, b));
      tf_store(next, out);
      tf_apply(next, in + 19, out + 12);
      break;
    }
    case OP_TIME_DIFF: {
      const RosDuration d = ros_time_diff((uint32_t)in[0], (uint32_t)in[1], (uint32_t)in[2], (uint32_t)in[3]);
      out[0] = d.sec; out[1] = d.nsec;
      out[2] = ros_duration_to_sec(d);
      out[3] = ros_time_to_sec((uint32_t)in[0], (uint32_t)in[1]);
      break;
    }
    case OP_FROM_SEC: {
      const RosDuration d = ros_duration_from_sec(in[0]);
      out[0] = d.sec; out[1] = d.nsec;
      out[2] = ros_duration_to_sec(d);
      break;
    }
    case OP_DURATION_GT: {
      const RosDuration a = ros_duration_from_sec(in[0]), b = ros_duration_from_sec(in[1]);
      out[0] = ros_duration_gt(a, b); out[1] = ros_duration_gt(b, a);
      break;
    }
    case OP_SET_RPY: quat_set_rpy(in[0], in[1], in[2], out); break;
    case OP_GET_RPY:
      tf_identity(t);
      for (int i = 0; i < 9; i++) t.m[i / 3][i % 3] = in[i];
      tf_get_rpy(t, out[0], out[1], out[2]);
      break;
    case OP_TF_GET_YAW: out[0] = tf_get_yaw(in); break;
    case OP_TF2_GET_YAW: out[0] = tf2_get_yaw(in); break;
    case OP_KROUND: out[0] = kround(in[0]); break;
    case OP_CAST_I32: out[0] = cast_i32(in[0]); break;
    case OP_CAST_U32: out[0] = cast_u32(in[0]); break;
    case OP_NORMALIZE_ANGLE: out[0] = normalize_angle(in[0]); break;
    case OP_NORMALIZE_DIFF: out[0] = normalize_angle_difference(in[0], in[1]); break;
    case OP_WORLD_TO_GRID: out[0] = world_to_grid_1(in[0], in[1], in[2]); break;
    case OP_N_STEPS: out[0] = n_steps(in[0], in[1]); break;
    case OP_SENSOR_POSE: sensor_pose_of(in, in + 3, out); break;
  }
}

__global__ void k_records(const Rec *__restrict__ recs, int n, double *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) eval_op(recs[i], out + (size_t)i * NOUT);
}

struct Records {
  std::vector<Rec> recs;
  std::map<std::string, long> branches;
  void push(int op, std::initializer_list<double> in) { push(op, std::vector<double>(in).data()); }
  void push(int op, const double *in) {
    Rec r{};
    r.op = op;
    for (int k = 0; k < OP_N_IN[op]; k++) r.in[k] = in[k];
    recs.push_back(r);
  }
  std::vector<double> host(int op, const double *in) {
    Rec r{};
    r.op = op;
    for (int k = 0; k < OP_N_IN[op]; k++) r.in[k] = in[k];
    std::vector<double> out(NOUT);
    eval_op(r, out.data());
    return out;
  }

  // the ros_math sweep's sink: each function on its inputs, later stages fed with the host build's results
  void rotation(const double m[9]) {
    const double trace = m[0] + m[4] + m[8];
    branches[trace > 0.0 ? "get_rotation_trace" : m[0] < m[4] ? (m[4] < m[8] ? "get_rotation_i2" : "get_rotation_i1")
                                                              : (m[0] < m[8] ? "get_rotation_i2" : "get_rotation_i0")]++;
    push(OP_GET_ROTATION, m);
    branches[std::fabs(m[6]) >= 1 ? (m[6] > 0 ? "get_rpy_singular_up" : "get_rpy_singular_down") : "get_rpy"]++;
    push(OP_GET_RPY, m);
    const std::vector<double> q = host(OP_GET_ROTATION, m);
    const double sarg = -2 * (q[0] * q[2] - q[3] * q[1]) / (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    branches[sarg <= -0.99999 ? "tf2_yaw_sarg_low" : sarg >= 0.99999 ? "tf2_yaw_sarg_high" : "tf2_yaw"]++;
    push(OP_TF2_GET_YAW, q.data());
  }
  void quaternion(const double q[4]) {
    push(OP_SET_ROTATION, q);
    push(OP_TF_GET_YAW, q);
    rotation(host(OP_SET_ROTATION, q).data());
  }
  void rpy(double r, double p, double y) {
    const double in[3] = {r, p, y};
    push(OP_SET_RPY, in);
    quaternion(host(OP_SET_RPY, in).data());
  }
  void entries(const double m[3][3], const double o[3]) { rotation(&m[0][0]); }
  void chain(const double q[4], const double o[3], const double q2[][4], const double o2[][3], const double v[][3]) {
    std::vector<double> acc = host(OP_SET_ROTATION, q);
    for (int i = 0; i < 3; i++) acc[9 + i] = o[i];
    for (int step = 0; step < ROS_MATH_CHAIN_STEPS; step++) {
      double in[23];
      for (int k = 0; k < 12; k++) in[k] = acc[k];
      for (int k = 0; k < 4; k++) in[12 + k] = q2[step][k];
      for (int k = 0; k < 3; k++) in[16 + k] = o2[step][k], in[19 + k] = v[step][k];
      in[22] = step % 3;
      push(OP_CHAIN_STEP, in);
      acc = host(OP_CHAIN_STEP, in);
      rotation(acc.data());
    }
  }
  void stamps(uint32_t s1, uint32_t n1, uint32_t s0, uint32_t n0) {
    branches[(int64_t)(int32_t)n1 - (int32_t)n0 < 0 ? "time_diff_nsec_negative" : "time_diff_nsec_positive"]++;
    if ((int64_t)(int32_t)s1 - (int32_t)s0 != (int32_t)(s1 - s0)) branches["time_diff_sec_wraps"]++;
    push(OP_TIME_DIFF, {(double)s1, (double)n1, (double)s0, (double)n0});
  }
  void from_sec(double d) {
    if (std::round((d - std::floor(d)) * 1e9) >= 1e9) branches["from_sec_rollover"]++;
    if (d < 0) branches["from_sec_negative"]++;
    push(OP_FROM_SEC, {d});
  }
  void from_sec_pair(double d, double d2) {
    from_sec(d);
    push(OP_DURATION_GT, {d, d2});
  }
};

// Math.h's math::Round as written: the form kround restates
double math_h_round(double v) { return v >= 0.0 ? floor(v + 0.5) : ceil(v - 0.5); }

void common_inputs(Records &R) {
  std::vector<double> scalars = {0.0, -0.0, NAN, -NAN, INFINITY, -INFINITY, 1e-300, -1e-300, 4.9e-324, -4.9e-324,
                                 0.49999999999999994, -0.49999999999999994, 2147483647.0, 2147483647.5,
                                 2147483648.0, -2147483648.0, -2147483648.5, -2147483649.0, 4294967295.0,
                                 4294967295.5, 4294967296.0, 9223372036854775808.0, -9223372036854775808.0,
                                 4503599627370495.5, 4503599627370496.0, -4503599627370495.5, 1e6, -1e6, 1e300};
  for (int k = -64; k <= 64; k++)  // half-integer ties and their neighbours
    for (double v : {k + 0.5, (double)k}) scalars.insert(scalars.end(), {v, std::nextafter(v, 1e300), std::nextafter(v, -1e300)});
  for (double e : {2147483648.0, 9223372036854775808.0})  // the int32 / int64 range edges, both signs, +-1 ulp
    for (double sg : {1.0, -1.0})
      for (double v : {sg * e, std::nextafter(sg * e, 0.0), std::nextafter(sg * e, sg * 1e300)}) scalars.push_back(v);
  for (double v : scalars) {
    R.push(OP_KROUND, {v});
    R.push(OP_CAST_I32, {v});
    R.push(OP_CAST_U32, {v});
  }
  // angles: +-1e6 rad and the wrap points; normalize_angle needs a finite angle (it loops on an infinite one)
  std::vector<double> angles = {0.0, -0.0, KT_PI, -KT_PI, std::nextafter(KT_PI, 4.0), std::nextafter(-KT_PI, -4.0),
                                KT_2PI, -KT_2PI, std::nextafter(KT_2PI, 7.0), std::nextafter(-KT_2PI, -7.0), 3 * KT_PI,
                                -3 * KT_PI, 1e6, -1e6, 999999.5, -123456.789, 1e-300};
  for (int k = 0; k < 2000; k++) angles.push_back(std::ldexp(std::sin(k * 12.9898) * 43758.5453, -(k % 20)));
  for (double a : angles) R.push(OP_NORMALIZE_ANGLE, {a});
  for (size_t i = 0; i + 1 < angles.size(); i++) R.push(OP_NORMALIZE_DIFF, {angles[i], angles[i + 1] * 0.5});
  // WorldToGrid at half-cell boundaries (+-1 ulp) for the resolutions the tests use, and the search step counts
  for (double res : {0.01, 0.02, 0.025, 0.03, 0.05, 0.1, 0.5})
    for (double off : {0.0, -10.0, -12.345, 3.3, -51.2}) {
      const double scale = 1.0 / res;
      for (int k = -60; k <= 60; k++) {
        const double w = off + (k + 0.5) * res;
        for (double x : {w, std::nextafter(w, 1e300), std::nextafter(w, -1e300), off + k * res})
          R.push(OP_WORLD_TO_GRID, {x, off, scale});
      }
      for (int k = 0; k < 40; k++) R.push(OP_N_STEPS, {k * res * 0.25, res});
      for (double s : {0.3, 0.5, 0.075, 0.35, 1.0}) R.push(OP_N_STEPS, {s, res});
    }
  // GetSensorAt: robot poses (zero, ordinary, heading +-1e6 rad) and laser offsets
  for (int k = 0; k < 3000; k++) {
    const double h = std::sin(k * 78.233) * 43758.5453, f = h - std::floor(h);
    const double th = k % 7 == 0 ? (k % 2 ? 1e6 : -1e6) + f : (f * 2 - 1) * (k % 3 == 0 ? 20.0 : KT_PI);
    const double robot[3] = {k % 11 == 0 ? 0.0 : (f - 0.5) * 40, k % 11 == 0 ? 0.0 : std::cos(k * 1.7) * 30,
                             k % 11 == 0 ? 0.0 : th};
    const double offset[3] = {std::cos(k * 0.37) * 0.5, std::sin(k * 0.91) * 0.3, std::sin(k * 0.13) * 3.2};
    R.push(OP_SENSOR_POSE, {robot[0], robot[1], robot[2], offset[0], offset[1], offset[2]});
  }
}

std::string rec_hex(const Rec &r) {
  std::string s = OP_NAMES[r.op];
  for (int k = 0; k < OP_N_IN[r.op]; k++) s += (k ? "," : ":") + hex64(r.in[k]);
  return s;
}

void groups_records(bool host_only, const std::string &out_dir) {
  Records R;
  ros_math_sweep(R);
  common_inputs(R);
  const int n = (int)R.recs.size();
  std::vector<double> host((size_t)n * NOUT), dev((size_t)n * NOUT, NAN);
  parallel_for((size_t)n, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; i++) eval_op(R.recs[i], &host[i * NOUT]);
  });
  if (!host_only) {
    Rec *d_recs = nullptr;
    double *d_out = nullptr;
    CK(cudaMalloc(&d_recs, n * sizeof(Rec)));
    CK(cudaMalloc(&d_out, dev.size() * sizeof(double)));
    CK(cudaMemcpy(d_recs, R.recs.data(), n * sizeof(Rec), cudaMemcpyHostToDevice));
    k_records<<<(n + 127) / 128, 128>>>(d_recs, n, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(dev.data(), d_out, dev.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CK(cudaFree(d_recs));
    CK(cudaFree(d_out));
  }
  // bit-identical groups, and the device / host difference counts of the libm ones
  std::map<std::string, long> inputs, differ;
  std::map<std::string, Misses> miss;
  std::map<std::string, long> per_op;
  long kround_vs_math_h = 0;
  std::string kround_first;
  FILE *bin = std::fopen((out_dir + "/libm_records.bin").c_str(), "wb");
  if (!bin) { std::fprintf(stderr, "cannot write %s/libm_records.bin\n", out_dir.c_str()); std::exit(2); }
  for (int i = 0; i < n; i++) {
    const Rec &r = R.recs[i];
    const std::string g = op_group(r.op);
    inputs[g]++;
    per_op[OP_NAMES[r.op]]++;
    if (r.op == OP_KROUND && !same_d(host[(size_t)i * NOUT], math_h_round(r.in[0])) && !kround_vs_math_h++)
      kround_first = rec_hex(r);
    bool d = false;
    for (int k = 0; k < NOUT; k++) d |= !same_d(dev[(size_t)i * NOUT + k], host[(size_t)i * NOUT + k]);
    if (op_is_libm(r.op)) {
      double row[18];
      row[0] = r.op;
      for (int k = 0; k < 9; k++) row[1 + k] = k < OP_N_IN[r.op] ? r.in[k] : 0.0;
      for (int k = 0; k < 4; k++) row[10 + k] = dev[(size_t)i * NOUT + k], row[14 + k] = host[(size_t)i * NOUT + k];
      std::fwrite(row, sizeof row, 1, bin);
      differ[g] += d && !host_only;
    } else if (d && !host_only) {
      miss[g].add(rec_hex(r));
    }
  }
  std::fclose(bin);
  for (const char *g : {"ros_math_arith", "ros_math_libm", "common_helpers"}) {
    std::printf("{\"group\": \"%s\", \"host_only\": %s, \"inputs\": %ld, \"mismatches\": %ld, \"first\": %s, "
                "\"device_host_differ_libm\": %ld",
                g, host_only ? "true" : "false", inputs[g], miss[g].n.load(), miss[g].json().c_str(), differ[g]);
    if (!std::strcmp(g, "common_helpers"))
      std::printf(", \"kround_vs_math_h\": %ld, \"kround_vs_math_h_first\": \"%s\"", kround_vs_math_h, kround_first.c_str());
    std::printf(", \"ops\": {");
    const char *sep = "";
    for (int op = 0; op < N_OPS; op++)
      if (op_group(op) == std::string(g)) {
        std::printf("%s\"%s\": %ld", sep, OP_NAMES[op], per_op[OP_NAMES[op]]);
        sep = ", ";
      }
    std::printf("}");
    if (std::string(g) != "common_helpers") {
      std::printf(", \"branches\": {");
      sep = "";
      for (const auto &b : R.branches) {
        std::printf("%s\"%s\": %ld", sep, b.first.c_str(), b.second);
        sep = ", ";
      }
      std::printf("}");
    }
    std::printf("}\n");
  }
  std::fflush(stdout);
}

}  // namespace

int main(int argc, char **argv) {
  bool host_only = false;
  std::string out_dir = ".";
  for (int i = 1; i < argc; i++) {
    if (!std::strcmp(argv[i], "--host-only")) host_only = true;
    else if (!std::strcmp(argv[i], "--out") && i + 1 < argc) out_dir = argv[++i];
  }
  const int variant = glibc_sincosf_variant_of_host();
  std::printf("{\"group\": \"setup\", \"host_variant\": %d, \"host_threads\": %d}\n", variant, n_threads());
  if (host_only) {
    group_sincosf_host(true);
    group_sincosf_host(false);
    groups_records(true, out_dir);
    return 0;
  }
  CK(cudaSetDevice(0));
  group_sincosf(true, variant);
  group_sincosf(false, variant);

  // Hector pose angles: util_normalize_angle keeps them in [-pi, pi], and one match moves them by at most 0.2 rad per
  // Gauss-Newton iteration (the clamp of dir[2]); the de-skew's yaw / pitch / roll are IMU angles integrated over one
  // scan.  |a| <= 16 covers 2 pi + 14 * 0.2 with room to spare.
  const Domain trig{0x41800000u, 0x41800000u};
  unsigned long long *d_sep = nullptr;
  CK(cudaMalloc(&d_sep, sizeof(unsigned long long)));
  CK(cudaMemset(d_sep, 0, sizeof(unsigned long long)));
  group_exhaustive(
      "hector_trig_exact", trig,
      [&](size_t base, size_t m, float2 *o) { k_trig_exact<<<(unsigned)((m + 255) / 256), 256>>>(trig, base, m, o, d_sep); },
      [](float a, float &s, float &c) { s = (float)sin((double)a); c = (float)cos((double)a); }, "separate_sin_cos_differ",
      d_sep);
  CK(cudaFree(d_sep));

  // log-odds cell values: every float in [-128, 64], including those below about -103.3 where the float odds underflow
  const Domain prob{0x42800000u, 0x43000000u};
  group_exhaustive(
      "hector_prob_exact", prob,
      [&](size_t base, size_t m, float2 *o) { k_prob_exact<<<(unsigned)((m + 255) / 256), 256>>>(prob, base, m, o); },
      [](float lo, float &odds, float &p) { odds = (float)exp((double)lo); p = log_odds_prob(lo); }, nullptr, nullptr);

  groups_records(false, out_dir);
  CK(cudaDeviceSynchronize());
  return 0;
}
