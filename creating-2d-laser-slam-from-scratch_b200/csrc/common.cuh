// Shared host/device helpers for libb200slam (sm_90a only).
//
// Arithmetic rule of this library: every double/float expression that feeds an integer grid index
// follows the reference's operation order with no FMA contraction (the library is compiled with
// -fmad=false and the critical expressions use explicit __dmul_rn/__dadd_rn), because the reference's
// x86-64 build has none either (SURVEY.md §7 "libm vs CUDA math").
#pragma once

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>

#include "../../include/b200slam.h"

namespace b2s {

void set_last_error(const std::string &s);
std::string &last_error_ref();

#define B2S_CUDA_CHECK(expr)                                                                          \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) {                                                                          \
      ::b2s::set_last_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" +        \
                            __FILE__ + ":" + std::to_string(__LINE__) + ")");                         \
      return B2S_ERR_CUDA;                                                                            \
    }                                                                                                 \
  } while (0)

#define B2S_FAIL(code, msg)        \
  do {                             \
    ::b2s::set_last_error(msg);    \
    return (code);                 \
  } while (0)

// ---- owners of the library's CUDA resources.  Every allocation, stream and event a handle or a call makes is held by
// one of these, so error paths release what they made by returning.  Destructors ignore CUDA return codes and never
// write the last-error text: the error already recorded is the one to report.

// device memory (cudaMalloc), or pinned host memory (cudaHostAlloc) when HOST.  reserve(n) grows only: the contents are
// discarded and at least one element is allocated.  With cudaHostAllocMapped, `dev` is the device alias of the memory.
template <class T, bool HOST = false>
struct Buf {
  T *p = nullptr, *dev = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf &operator=(Buf &&o) noexcept {  // a swap: the old memory goes with `o`
    std::swap(p, o.p);
    std::swap(dev, o.dev);
    std::swap(cap, o.cap);
    return *this;
  }
  ~Buf() { reset(); }
  operator T *() const { return p; }
  cudaError_t reset() {
    T *q = p;
    p = dev = nullptr;
    cap = 0;
    return !q ? cudaSuccess : HOST ? cudaFreeHost((void *)q) : cudaFree((void *)q);
  }
  cudaError_t reserve(size_t n, unsigned host_flags = cudaHostAllocDefault) {
    n = std::max<size_t>(n, 1);
    if (p && n <= cap) return cudaSuccess;
    if (cudaError_t e = reset()) return e;
    void *q = nullptr;
    cudaError_t e = HOST ? cudaHostAlloc(&q, n * sizeof(T), host_flags) : cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess) return e;
    p = static_cast<T *>(q);
    cap = n;
    if (host_flags & cudaHostAllocMapped) {
      void *d = nullptr;
      if ((e = cudaHostGetDevicePointer(&d, q, 0)) != cudaSuccess) return e;
      dev = static_cast<T *>(d);
    }
    return cudaSuccess;
  }
};
template <class T>
using HostBuf = Buf<T, true>;

// stream-ordered memory of one call: cudaMallocAsync, and cudaFreeAsync on the same stream at scope exit
template <class T>
struct AsyncBuf {
  T *p = nullptr;
  cudaStream_t s;
  explicit AsyncBuf(cudaStream_t stream) : s(stream) {}
  AsyncBuf(const AsyncBuf &) = delete;
  AsyncBuf &operator=(const AsyncBuf &) = delete;
  ~AsyncBuf() {
    if (p) cudaFreeAsync(p, s);
  }
  operator T *() const { return p; }
  cudaError_t alloc(size_t n) { return cudaMallocAsync(reinterpret_cast<void **>(&p), n * sizeof(T), s); }
};

struct Event {
  cudaEvent_t e = nullptr;
  Event() = default;
  Event(const Event &) = delete;
  Event &operator=(const Event &) = delete;
  ~Event() {
    if (e) cudaEventDestroy(e);
  }
  operator cudaEvent_t() const { return e; }
  cudaError_t create(unsigned flags = cudaEventDefault) { return cudaEventCreateWithFlags(&e, flags); }
};

// the caller's stream, borrowed; or, when the caller passes none, a non-blocking stream created and destroyed here.
// Handles declare it first, so that it is destroyed after everything else they own.
struct Stream {
  cudaStream_t s = nullptr;
  bool owned = false;
  Stream() = default;
  Stream(const Stream &) = delete;
  Stream &operator=(const Stream &) = delete;
  ~Stream() {
    if (owned) cudaStreamDestroy(s);
  }
  operator cudaStream_t() const { return s; }
  cudaError_t init(void *borrowed) {
    if (borrowed) {
      s = reinterpret_cast<cudaStream_t>(borrowed);
      return cudaSuccess;
    }
    const cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    owned = e == cudaSuccess;
    return e;
  }
};

constexpr double KT_PI = 3.14159265358979323846;   // Math.h:32
constexpr double KT_2PI = 6.28318530717958647692;  // Math.h:33
constexpr double KT_TOLERANCE = 1e-06;             // Math.h:41
constexpr int32_t INVALID_SCAN = 2147483647;       // Math.h:47
constexpr int GRID_OCCUPIED = 100;                 // Karto.h:4196
constexpr int GRID_FREE = 255;                     // Karto.h:4197
constexpr double MAX_VARIANCE = 500.0;             // Mapper.cpp:36
constexpr double DISTANCE_PENALTY_GAIN = 0.2;      // Mapper.cpp:37
constexpr double ANGLE_PENALTY_GAIN = 0.2;         // Mapper.cpp:38

// math::Round (Math.h:87-90): half away from zero, v >= 0 ? floor(v + 0.5) : ceil(v - 0.5).  The same bits with one
// rounding op instead of two: ceil(v - 0.5) == -floor(-v + 0.5) for v < 0 (negation is exact), and -0.0 takes the
// v >= 0 side to +0.0 (tests/device_math_check.cu compares both builds with the reference's form).
__host__ __device__ __forceinline__ double kround(double v) {
  const double r = floor(fabs(v) + 0.5);
  return v < 0.0 ? -r : r;
}

// static_cast<kt_int32s>(double) as the reference's x86-64 build performs it (cvttsd2si: out-of-range and NaN
// give INT_MIN); CUDA's own conversion saturates instead.
__host__ __device__ __forceinline__ int32_t cast_i32(double d) {
  return (d >= -2147483648.0 && d < 2147483648.0) ? (int32_t)d : (int32_t)0x80000000;
}
// static_cast<kt_int32u>(double): cvttsd2si 64-bit then truncation
__host__ __device__ __forceinline__ uint32_t cast_u32(double d) {
  return (d >= -9223372036854775808.0 && d < 9223372036854775808.0) ? (uint32_t)(long long)d : 0u;
}

// math::DoubleEqual (Math.h:135-139)
__host__ __device__ __forceinline__ bool double_equal(double a, double b) {
  double delta = a - b;
  return delta < 0.0 ? delta >= -KT_TOLERANCE : delta <= KT_TOLERANCE;
}

// math::NormalizeAngle (Math.h:182-211)
__host__ __device__ inline double normalize_angle(double angle) {
  while (angle < -KT_PI) {
    if (angle < -KT_2PI)
      angle += (double)cast_u32(angle / -KT_2PI) * KT_2PI;
    else
      angle += KT_2PI;
  }
  while (angle > KT_PI) {
    if (angle > KT_2PI)
      angle -= (double)cast_u32(angle / KT_2PI) * KT_2PI;
    else
      angle -= KT_2PI;
  }
  return angle;
}

// math::NormalizeAngleDifference (Math.h:221-234)
__host__ __device__ inline double normalize_angle_difference(double minuend, double subtrahend) {
  while (minuend - subtrahend < -KT_PI) minuend += KT_2PI;
  while (minuend - subtrahend > KT_PI) minuend -= KT_2PI;
  return minuend;
}

__host__ __device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }  // math::Maximum

// CoordinateConverter::WorldToGrid, one axis (Karto.h:4237-4252)
__host__ __device__ __forceinline__ int32_t world_to_grid_1(double w, double offset, double scale) {
  return cast_i32(kround((w - offset) * scale));
}

// number of search steps: static_cast<kt_int32u>(math::Round(off * 2.0 / res) + 1) (Mapper.cpp:339-341,361)
__host__ __device__ __forceinline__ int n_steps(double off, double res) {
  return (int)cast_u32(kround(off * 2.0 / res) + 1);
}

// LocalizedRangeScan::GetSensorAt = Transform(robot).TransformPose(offset) (Karto.h:5310-5313, 2860-2935,
// Matrix3::FromAxisAngle 2392-2421 with axis (0,0,1), Matrix3*Pose2 2574-2583)
__host__ __device__ inline void sensor_pose_of(const double robot[3], const double offset[3], double out[3]) {
  double m00, m01, m02, m10, m11, m12, tx, ty, th;
  if (robot[0] == 0.0 && robot[1] == 0.0 && robot[2] == 0.0) {  // rPose1 == rPose2 (Karto.h:2911-2917)
    m00 = 1; m01 = 0; m02 = 0; m10 = 0; m11 = 1; m12 = 0; tx = 0; ty = 0; th = 0;
  } else {
    double radians = robot[2] - 0.0;
    double c = cos(radians), s = sin(radians), omc = 1.0 - c;
    m00 = 0.0 * omc + c;
    m01 = 0.0 * 0.0 * omc - 1.0 * s;
    m02 = 0.0 * 1.0 * omc + 0.0 * s;
    m10 = 0.0 * 0.0 * omc + 1.0 * s;
    m11 = 0.0 * omc + c;
    m12 = 0.0 * 1.0 * omc - 0.0 * s;
    tx = robot[0]; ty = robot[1]; th = robot[2] - 0.0;
  }
  double rx = m00 * offset[0] + m01 * offset[1] + m02 * offset[2];
  double ry = m10 * offset[0] + m11 * offset[1] + m12 * offset[2];
  out[0] = tx + rx;
  out[1] = ty + ry;
  out[2] = normalize_angle(offset[2] + th);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is one value per (kernel, device), shared by every handle of the process.
// Handles of different sizes used from different threads must therefore never LOWER it between another thread's set
// and launch: keep a process-wide running maximum per (kernel, device) and only ever raise the attribute.
template <class K>
inline cudaError_t raise_dyn_smem(K kern, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void *, int>, size_t> seen;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  size_t &cur = seen[std::make_pair(reinterpret_cast<const void *>(kern), dev)];
  if (bytes <= cur) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) cur = bytes;
  return e;
}

// Calls that stage through cudaMallocAsync / cudaFreeAsync and then synchronise would hand their memory back to the driver
// every time (the default pool's release threshold is 0) and pay a fresh allocation on the next call (~1 ms).  The
// library's create functions raise the threshold of the device's default pool once, so freed blocks stay cached.
inline void keep_pool_memory(int device) {
  static std::mutex mu;
  static std::map<int, bool> done;
  std::lock_guard<std::mutex> lock(mu);
  if (done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long keep = 1ull << 32;  // up to 4 GiB of freed staging blocks stay in the pool
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  cudaGetLastError();
  done[device] = true;
}

inline b2s_status check_device(int device) {
  if (b2s_device_count() <= device) B2S_FAIL(B2S_ERR_NO_DEVICE, "no usable CUDA device (the product path has no CPU fallback)");
  return B2S_OK;
}

// prologue of every entry point that creates device state
inline b2s_status open_device(int device) {
  if (b2s_status st = check_device(device)) return st;
  B2S_CUDA_CHECK(cudaSetDevice(device));
  keep_pool_memory(device);
  return B2S_OK;
}

// NVTX range around a host entry point (SURVEY.md §5 tracing): shows up as "b2s:<name>" in Nsight timelines; nvtx3 is
// header-only and costs a predictable branch when no tool is attached.
struct NvtxRange {
  explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange &) = delete;
  NvtxRange &operator=(const NvtxRange &) = delete;
};
#define B2S_NVTX(name) ::b2s::NvtxRange _b2s_nvtx_range("b2s:" name)

// ---- mbarrier (shared-memory transaction barrier) wrappers: the Karto window sweep waits on its TMA copies with them,
// the Hector cluster match on the partial sums its peers send ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// true once the phase of `parity` has completed; the instruction itself suspends the thread for a while before it says no
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// gridDim.y's limit.  Kernels that put a batch on grid y loop `for (b = blockIdx.y; b < count; b += gridDim.y)` and are
// launched with grid_rows(count) rows, so a batch of any size runs; up to this many items each row serves one.
constexpr int GRID_Y_MAX = 65535;
inline unsigned grid_rows(long long count) { return (unsigned)std::min<long long>(std::max<long long>(count, 1), GRID_Y_MAX); }

// SMs of `device` (132 on an H100 SXM): grid-stride kernels size their grids as a multiple of it.
inline int sm_count(int device) {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms < 1) {
    cudaGetLastError();
    sms = 1;
  }
  return sms;
}

}  // namespace b2s
