// lesson4 front end — hectorslam::HectorSlamProcessor on H100 (sm_90a).  Product code: CUDA only.
//
// Reference behaviour (paths relative to reference/lesson4/include/lesson4/hector_mapping):
//   HectorSlamProcessor::update / reset                                  slam_main/HectorSlamProcessor.h:81-116
//   MapRepMultiMap ctor / matchData / updateByScan                       slam_main/MapRepMultiMap.h:56-191
//   ScanMatcher::matchData / estimateTransformationLogLh                 matcher/ScanMatcher.h:60-141
//   OccGridMapUtil::getCompleteHessianDerivs / interpMapValueWithDerivatives / getTransformForState
//                                                                        map/OccGridMapUtil.h:77-228, 437-440
//   OccGridMapBase::updateByScan / Bresenham / bresenhamCellFree/Occ     map/OccGridMapBase.h:118-168, 220-330
//   GridMapLogOddsFunctions::getGridProbability                          map/GridMapLogOdds.h:136-140
//   util::poseDifferenceLargerThan / normalize_angle                     util/UtilFunctions.h:36-48, 72-90
//   node loop: update(container, getLastScanMatchPose())                 lesson4/src/hector_mapping/hector_slam.cc:195-204
//
// Everything of one LaserScan runs on the device: the coarse-to-fine Gauss-Newton match, the map-update gate, the
// pose -> cell transform of the update and the Bresenham mark / apply passes.  The processor's state (last poses,
// update indices, stamp epochs, the coarse levels' data containers) lives in device memory, so a stream of scans needs
// no host round trip between scans (b2s_hector_slam_process_stream: ONE cooperative kernel walks the whole stream;
// b2s_hector_slam_update: one launch per scan, the pose comes back through a host-mapped mailbox as soon as the match
// is done while the map update still runs).  A handle holds B independent processors (independent robots / maps,
// SURVEY.md §8(e): "shard over independent maps"), each with its own map layout and settings (one HsProc row of a
// device table; b2s_hector_slam_create_fleet); B = 1 is the reference's single processor.  They step together one
// scan each (b2s_hector_slam_update_batch: three launches per step), or each walks its own recording in ONE launch, one
// CTA per processor (b2s_hector_slam_process_stream_batch; b2s_hector_slam_process_scans_batch takes the raw LaserScan
// ranges and converts each scan inside that launch).
//
// Arithmetic: float32 in the reference's operation order, no FMA (-fmad=false).  EXACT mode (default) reproduces the
// reference bit for bit: the nine sums of getCompleteHessianDerivs are accumulated sequentially in point order (one lane
// per sum), Rotation2Df's std::cos / std::sin(float) are glibc's sincosf restated (glibc_math.cuh), the unqualified
// sin / cos / exp of the reference (C library DOUBLE functions rounded to float) are the device's double functions
// rounded to float (libm_sincos_to_float, log_odds_prob).  Those floats equal glibc's for EVERY float angle with
// |a| <= 16 and every float log-odds value in [-128, 64]: tests/test_gpu_device_math.py compares all of them.  FAST mode differs in ONE thing: the nine sums are
// tree-reduced (warp shuffles) instead of accumulated in point order, so its Hessians / poses differ in the last float bits
// (~1e-6 m per scan, inside the 1e-4 contract) and a cell can move when a pose lands an ulp away.
//
// The grid arithmetic it shares with the single-map handle (hector_map.cu) is in hector_grid.cuh: map transform, begin /
// end cells, Bresenham set-up and step, bilinear bounds test and finish, 3x3 solve, normalize_angle, ROS map, log-odds
// factors.  Its own: the pyramid, the probability quads (double exp), 32-bit stamps with the bounding-box apply sweep,
// the begin cell on the device, and the match's two-halves fetch.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"
#include "glibc_math.cuh"
#include "hector_grid.cuh"
#include "hector_node_plan.cuh"
#include "hector_scan.cuh"

using namespace b2s;

namespace b2s {

constexpr int HS_L = B2S_HECTOR_MAX_LEVELS;
constexpr int HS_THREADS = 576;          // 18 warps: two points per thread cover a 1081-beam scan in one pass
constexpr int HS_MAX_PTS = 4096;         // beams per scan (12-bit beam field of the stamps; shared-memory staging)
constexpr int HS_EPOCH_BITS = 20;
constexpr unsigned HS_EPOCH_MAX = (1u << HS_EPOCH_BITS) - 1;
constexpr int HS_STREAM_CTAS = 48;       // cooperative grid of the stream kernel (one CTA per SM, all co-resident)

struct HsLevel {  // one MapRepMultiMap level of ONE processor: its planes, already offset into the level's pools
  float4 *quad;   // per cell (x, y): getGridProbability of the four cells (x, y), (x+1, y), (x, y+1), (x+1, y+1) — what one
                  // bilinear look-up of the matcher reads — refreshed whenever a cell's log-odds changes (the device-side
                  // form of the reference's per-scan GridMapCacheArray).  ONE 16-byte load per scan point instead of four
                  // scattered 4-byte ones: the match's per-point phase was bound by L1 tag throughput (gathers)
  float *lo;
  int32_t *ui;
  uint32_t *free_st, *occ_st;  // per-scan stamps: (epoch << 12) | (4095 - beam)
  float *pts;                  // [cap][2] data container of this level (level 0: the current scan)
  int sx, sy;
  MapTransform tf;
  int iterations;  // 1 + maxIterations of MapRepMultiMap::matchData (:144-166): 1+5 on level 0, 1+3 above
};

// One processor's map layout and settings: a row of the handle's device table (HsBatch::procs).  Every kernel copies
// its processor's row into shared memory first (hs_load_proc); levels at or above `levels` have no planes.
struct HsProc {
  HsLevel l[HS_L];
  int levels;
  float lo_free, lo_occ, min_dist, min_angle;
};

struct HsState {  // device-resident state of ONE processor
  float last_update_pose[3], last_match_pose[3], last_cov[9];
  int curr_update_index[HS_L];
  unsigned int epoch[HS_L];
  int n_pts[HS_L];
  float origo[HS_L][2];
  // the update the gate decided for the current scan
  int do_update;
  float uc[HS_L], us[HS_L], umx[HS_L], umy[HS_L];
  int bx[HS_L], by[HS_L];
  unsigned int epoch_hi[HS_L];
  int mark_free[HS_L], mark_occ[HS_L];
  int bb_x0[HS_L], bb_y0[HS_L], bb_x1[HS_L], bb_y1[HS_L];  // cells the update's rays can touch (inclusive; empty: x1 < x0)
  unsigned long long visits, n_matched, n_updated;
  unsigned long long t_match_ns, t_update_ns;
};

struct HsBatch {  // kernel parameter
  const HsProc *procs;  // [batch] device
  int batch, cap;
  int exact, use_fma;
  HsState *state;  // [batch]
};

// processor b's row of the table -> `dst` (shared memory), by the whole CTA; ends with a __syncthreads
__device__ __forceinline__ void hs_load_proc(const HsBatch &P, int b, HsProc *dst) {
  static_assert(sizeof(HsProc) % sizeof(int) == 0, "copied as words");
  const int *s = reinterpret_cast<const int *>(P.procs + b);
  int *d = reinterpret_cast<int *>(dst);
  for (int i = threadIdx.x; i < (int)(sizeof(HsProc) / sizeof(int)); i += blockDim.x) d[i] = s[i];
  __syncthreads();
}

struct HsCall {  // one scan per processor
  const float *pts0;    // [b][pts_stride][2] level-0 points (device, or host-mapped for the per-scan call)
  const int *n0;        // [b] (device / host-mapped) or NULL -> n0_uniform
  int n0_uniform, pts_stride;
  const float *hints;   // [b][3] or NULL -> the processor's last scan-match pose (the node's loop)
  float origo_x, origo_y;
  int map_without_matching;
  float *out;           // [b][16] device: pose[3], cov[9], updated, matched, exchange-lost, -
  volatile float *mailbox;  // host-mapped copy of out for processor 0 + sequence word, or NULL
  unsigned int seq;
  unsigned int tag;     // != 0: published (release, gpu scope) in out[b][15] once the scan's state is complete
  float *carry;         // shared-memory [3] or NULL: receives the scan-match pose (the next scan's hint in a stream)
  int own_row = 0;      // 0: row b of hints / out / n0 is processor b's; != 0: they already point at this CTA's scan
                        // (row 0), whatever b is — a processor walking its own stream (k_hs_stream_batch)
};

__device__ __forceinline__ unsigned long long hs_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- thread-block cluster exchange of the fast single-stream match (k_hs_stream<false, true>) ----
// The per-point phase of a Gauss-Newton iteration is issue-bound on ONE SM (most of the iteration's cycles), so the
// CTAs of cluster 0 split the scan's points: rank 0 (the master) solves, the helpers receive the pose + sine / cosine and
// return their nine partial sums through distributed shared memory.  Data and signal travel together (st.async with
// mbarrier complete_tx): no cluster-scope fence, hence no L1 invalidation (CCTL.IVALL) inside the iteration loop.
// (Tried and rejected: 8-byte {value, sequence} messages written with plain st.shared::cluster and polled with volatile
// shared loads — no mbarrier at all — were slower per hop than st.async + try_wait.)
constexpr int HS_CLUSTER = 4;
constexpr int HS_POSE_WORDS = 7;  // e0, e1, cos, sin, sinRot, cosRot, spare
struct __align__(16) HsXchg {
  uint64_t bar_pose, bar_part;  // mbarriers: pose arrived (helpers) / all partial sums arrived (master)
  float pose[8];
  float part[HS_CLUSTER][12];             // [rank][sum]
};
__device__ __forceinline__ uint32_t hs_cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t hs_cluster_size() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t hs_mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void hs_st_async(uint32_t remote_addr, float v, uint32_t remote_bar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(remote_addr),
               "r"(__float_as_uint(v)), "r"(remote_bar)
               : "memory");
}
// bounded: a lost exchange must not hang the device (the host reports B2S_ERR_CUDA when the flag is set)
__device__ __forceinline__ bool mbar_wait_bounded(uint64_t *bar, uint32_t parity) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > (1ll << 25)) return false;  // ~17 ms; a legitimate wait is microseconds
  return true;
}
__device__ __forceinline__ void hs_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the points [p0, p1) of rank r when n points are split over `size` CTAs
__device__ __forceinline__ void hs_share(int n, int rank, int size, int &p0, int &p1) {
  const int chunk = (n + size - 1) / size;
  p0 = min(n, rank * chunk);
  p1 = min(n, p0 + chunk);
}

// interpMapValueWithDerivatives (OccGridMapUtil.h:139-228) in two halves so that the four cell loads of SEVERAL points are
// in flight together.  Plain loads (L1): within one launch the planes are only rewritten by the update passes, and every
// CTA passes the grid barrier's gpu-scope acquire (which drops the SM's L1 lines) between an update and the next match.
struct HsFetch {
  float i0, i1, i2, i3, fx, fy;
  bool inside;
};
__device__ __forceinline__ HsFetch hs_fetch(const float4 *__restrict__ quad, int sx, int sy, float x, float y) {
  HsFetch f;
  f.inside = interp_inside(sx, sy, x, y);
  f.i0 = f.i1 = f.i2 = f.i3 = 0.0f; f.fx = f.fy = 0.0f;
  if (f.inside) {
    const int ix = (int)x, iy = (int)y;
    f.fx = x - (float)ix; f.fy = y - (float)iy;
    const float4 q = quad[iy * sx + ix];
    f.i0 = q.x; f.i1 = q.y; f.i2 = q.z; f.i3 = q.w;
  }
  return f;
}
__device__ __forceinline__ void hs_finish(const HsFetch &f, float out[3]) {
  if (!f.inside) { out[0] = out[1] = out[2] = 0.0f; return; }
  interp_finish(f.i0, f.i1, f.i2, f.i3, f.fx, f.fy, out);
}

// util::poseDifferenceLargerThan (UtilFunctions.h:72-90).  Only <cmath> is included there, so the unqualified
// abs(angleDiff) is int abs(int): the difference is truncated to an integer before the compare.
__device__ inline bool hs_pose_difference_larger_than(const float a[3], const float b[3], float dist_thresh,
                                                      float angle_thresh) {
  const float dx = a[0] - b[0], dy = a[1] - b[1];
  if (sqrtf(dx * dx + dy * dy) > dist_thresh) return true;
  float d = a[2] - b[2];
  const double pi = 3.14159265358979323846;
  if ((double)d > pi) d = (float)((double)d - pi * 2.0f);
  else if ((double)d < -pi) d = (float)((double)d + pi * 2.0f);
  const int t = (int)d;
  return (float)(t < 0 ? -t : t) > angle_thresh;
}

// terms of one point for getCompleteHessianDerivs (OccGridMapUtil.h:99-126)
__device__ __forceinline__ HsFetch hs_point_fetch(const float4 *__restrict__ prob, int sx, int sy, float2 p, float c, float s,
                                                  float e0, float e1) {
  const float tx = (c * p.x + (-s) * p.y) + e0, ty = (s * p.x + c * p.y) + e1;
  return hs_fetch(prob, sx, sy, tx, ty);
}
__device__ __forceinline__ void hs_point_terms(const HsFetch &f, float2 p, float sin_rot, float cos_rot, float a[9]) {
  float t[3];
  hs_finish(f, t);
  const float rot = ((-sin_rot * p.x - cos_rot * p.y) * t[1] + (cos_rot * p.x - sin_rot * p.y) * t[2]);
  const float fun = 1.0f - t[0];
  a[0] = t[1] * fun; a[1] = t[2] * fun; a[2] = rot * fun;    // dTr
  a[3] = t[1] * t[1]; a[4] = t[2] * t[2]; a[5] = rot * rot;  // H00 H11 H22
  a[6] = t[1] * t[2]; a[7] = t[1] * rot; a[8] = t[2] * rot;  // H01 H02 H12
}

struct HsTrig {
  float c, s;              // Rotation2Df(angle): std::cos / std::sin(float) = glibc cosf / sinf
  float sin_rot, cos_rot;  // OccGridMapUtil.h:87-88: the C library's double sin / cos, rounded to float
};
// (out of line on purpose: the Gauss-Newton loop is executed by few warps, so its code must stay inside the instruction
// cache — 60-90 KB kernels with the double-precision sincos / fmod expansions inlined at every use ran markedly slower)
__device__ __noinline__ HsTrig hs_trig(float angle, bool exact, bool use_fma) {
  HsTrig t;
  if (exact) {
    glibc_sincosf(angle, use_fma, &t.s, &t.c);
    libm_sincos_to_float(angle, &t.sin_rot, &t.cos_rot);
  } else {
    // fast mode: the glibc-exact float sine / cosine also stand in for sinRot / cosRot (they differ from the rounded
    // double ones on ~1 % of angles, by one ulp).  The device's own sincosf was tried here and broke the 1e-4 contract on
    // one scan of the test stream: a few Gauss-Newton iterations amplify an ulp of the rotation noticeably.
    glibc_sincosf(angle, use_fma, &t.s, &t.c);
    t.sin_rot = t.s;
    t.cos_rot = t.c;
  }
  return t;
}

// Fast mode, cluster variant: the per-point phase of this CTA's share (points [0, cnt) of `pts`) and the CTA's nine sums.
// The phase is ISSUE-bound (one SM retires ~500 warp instructions per warp and iteration in the two-points-per-thread
// form), so: only the warps that own points run it, every thread stores its nine terms as columns (9 STS instead of a
// 45-shuffle tree per warp), and warps 0..8 then sum one column each.  Returns sum `warp` in every lane of warps 0..8.
// Contains one __syncthreads.
__device__ __forceinline__ float hs_share_sums(const float4 *__restrict__ prob, int sx, int sy, const float2 *pts, int cnt,
                                               float factor, float e0, float e1, float c, float s, float sin_rot,
                                               float cos_rot, float *terms, int pitch, int tid, int lane, int warp) {
  if (warp * 32 < cnt) {
#pragma unroll 1
    for (int i = tid; i < cnt; i += HS_THREADS) {
      const float2 p = make_float2(__fmul_rn(pts[i].x, factor), __fmul_rn(pts[i].y, factor));
      const HsFetch f = hs_point_fetch(prob, sx, sy, p, c, s, e0, e1);
      float t[9];
      hs_point_terms(f, p, sin_rot, cos_rot, t);
#pragma unroll
      for (int q = 0; q < 9; q++) terms[q * pitch + i] = t[q];
    }
  }
  __syncthreads();
  float v = 0.0f;
  if (warp < 9) {
    const float *col = terms + warp * pitch;
    // (not unrolled on purpose: this runs once per iteration on cold instruction lines — the L0 instruction cache holds
    // ~6 KB and the iteration loop is larger — so executed code BYTES cost more than instructions)
    float v1 = 0.0f, v2 = 0.0f, v3 = 0.0f;  // four loads in flight: the loop is a latency chain, not a throughput one
    int i = lane;
#pragma unroll 1
    for (; i + 96 < cnt; i += 128) { v += col[i]; v1 += col[i + 32]; v2 += col[i + 64]; v3 += col[i + 96]; }
#pragma unroll 1
    for (; i < cnt; i += 32) v += col[i];
    v = (v + v1) + (v2 + v3);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  }
  return v;
}

// shared memory of the match: [cap] float2 staged scan, then (EXACT) 9 term columns of `pitch` floats / (FAST) per-warp partials
__host__ __device__ inline int hs_pitch(int cap) { return ((cap + 3) & ~3) + 4; }
__host__ __device__ inline size_t hs_terms_offset(int cap) { return (sizeof(float2) * (size_t)cap + 15) & ~(size_t)15; }  // float4 reads of the columns
__host__ __device__ inline size_t hs_smem_bytes(int cap) { return hs_terms_offset(cap) + sizeof(float) * 9 * (size_t)hs_pitch(cap) + 64; }

// MapRepMultiMap::matchData (:144-166) on every level, coarsest first, + the gate and the update parameters of
// HectorSlamProcessor::update (:81-108), by ONE CTA for processor b.
// Q = processor b's row of the table (shared memory).  Returns the gate's verdict (map update or not).
// INGEST (k_hs_stream_batch<_, true>): the container's origo is the processor's own, which the host wrote into
// st->origo[0] before the launch (hs_ingest_upload), not C's.
template <bool EXACT, bool CLUSTER, bool INGEST = false>
__device__ bool hs_match_cta(const HsBatch &P, const HsProc &Q, const HsCall &C, int b, unsigned char *smem, HsXchg *xc = nullptr,
                             uint32_t *xc_parity = nullptr) {
  static_assert(!(EXACT && CLUSTER), "the bit-exact sums are one sequential chain: nothing to split");
  HsState *st = P.state + b;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = HS_THREADS / 32;
  const int row = C.own_row ? 0 : b;  // row of C.hints / C.out / C.n0
  const int n = C.n0 ? C.n0[row] : C.n0_uniform;
  constexpr bool exact = EXACT;  // compile-time: each mode's kernel carries only its own code
  const bool use_fma = P.use_fma != 0;
  float2 *spts = reinterpret_cast<float2 *>(smem);
  float *terms = reinterpret_cast<float *>(smem + hs_terms_offset(P.cap));
  const int pitch = hs_pitch(P.cap);
  __shared__ float bc[8];    // estimate + trig published by the solving thread
  __shared__ float tot[9];
  __shared__ float s_world[3];
  __shared__ int s_do;
  __shared__ int s_bb[HS_L][4];
  __shared__ int s_lost;
  const uint32_t csize = CLUSTER ? hs_cluster_size() : 1u;
  uint32_t part_parity = CLUSTER ? *xc_parity : 0u;
  int my0 = 0, my1 = n;  // this CTA's share of the points in the per-point phase
  if (CLUSTER) hs_share(n, 0, (int)csize, my0, my1);
  if (CLUSTER && tid == 0) s_lost = 0;
  // master -> helpers: the pose of the next iteration (bc[0..6]) into every helper's HsXchg::pose; one st.async per lane
  // of warp 0 (the solving thread publishes nothing itself: 21 serial remote stores would sit on its critical path)
  auto publish = [&]() {
    if constexpr (CLUSTER) {
      const uint32_t a_pose = smem_u32(xc->pose), a_bar = smem_u32(&xc->bar_pose);
#pragma unroll 1
      for (uint32_t l = (uint32_t)lane; l + HS_POSE_WORDS < HS_POSE_WORDS * csize; l += 32) {
        const uint32_t r = 1 + l / HS_POSE_WORDS, q = l % HS_POSE_WORDS;
        hs_st_async(hs_mapa(a_pose + 4 * q, r), bc[q], hs_mapa(a_bar, r));
      }
    }
  };
  // state the serial tail needs, requested now so that the loads' latency hides behind the match (written last by this
  // same thread, or by an earlier kernel)
  float lup[3] = {0.0f, 0.0f, 0.0f}, lcov[9];
  unsigned long long n_matched0 = 0;
  if (tid == 0) {
    lup[0] = st->last_update_pose[0]; lup[1] = st->last_update_pose[1]; lup[2] = st->last_update_pose[2];
    n_matched0 = st->n_matched;
#pragma unroll
    for (int q = 0; q < 9; q++) lcov[q] = st->last_cov[q];
  }
  const unsigned long long t0 = hs_now_ns();
  const float2 *gp = reinterpret_cast<const float2 *>(C.pts0) + (size_t)b * C.pts_stride;
  for (int i = tid; i < n; i += HS_THREADS) {
    const float2 p = gp[i];
    spts[i] = p;
    reinterpret_cast<float2 *>(Q.l[0].pts)[i] = p;  // level-0 container for the update passes
  }
  if (tid == 0) {
    const float *h = C.hints ? C.hints + 3 * row : st->last_match_pose;
    s_world[0] = h[0]; s_world[1] = h[1]; s_world[2] = h[2];
  }
  __syncthreads();
  float world0 = s_world[0], world1 = s_world[1], world2 = s_world[2];
  bool any = false;
  if (!C.map_without_matching && n > 0) {
    float factor = 1.0f;
    for (int l = 1; l < Q.levels; l++) factor *= 0.5f;  // static_cast<float>(1.0 / pow(2.0, l)) is exactly 2^-l
    for (int lv = Q.levels - 1; lv >= 0; lv--, factor *= 2.0f) {
      const HsLevel &m = Q.l[lv];
      const float4 *prob = m.quad;
      if (lv > 0)  // dataContainers[lv-1].setFrom(dataContainer, 2^-lv) (DataPointContainer.h:46-59): exact scaling
        for (int i = tid; i < n; i += HS_THREADS)
          reinterpret_cast<float2 *>(m.pts)[i] = make_float2(__fmul_rn(spts[i].x, factor), __fmul_rn(spts[i].y, factor));
      if (tid == 0) {
        float e0, e1;
        get_map_coords(m.tf, world0, world1, e0, e1);
        const HsTrig tr = hs_trig(world2, exact, use_fma);
        bc[0] = e0; bc[1] = e1; bc[2] = world2; bc[3] = tr.c; bc[4] = tr.s; bc[5] = tr.sin_rot; bc[6] = tr.cos_rot;
      }
      if (CLUSTER && warp == 0) {
        __syncwarp();
        publish();
      }
      __syncthreads();
      for (int it = 0; it < m.iterations; it++) {
        const float e0 = bc[0], e1 = bc[1], c = bc[3], s = bc[4], sin_rot = bc[5], cos_rot = bc[6];
        if constexpr (CLUSTER) {
          float v = hs_share_sums(prob, m.sx, m.sy, spts, my1, factor, e0, e1, c, s, sin_rot, cos_rot, terms, pitch, tid, lane, warp);
          if (warp < 9) {
            if (csize > 1) {  // + the helpers' partial sums, in rank order
              if (tid == 0) mbar_expect_tx(&xc->bar_part, 36u * (csize - 1));
              if (!mbar_wait_bounded(&xc->bar_part, part_parity)) s_lost = 1;  // every reading thread observes the phase itself
#pragma unroll 1
              for (uint32_t r = 1; r < csize; r++) v += xc->part[r][warp];
            }
            if (lane == 0) tot[warp] = v;
          }
          if (csize > 1) part_parity ^= 1u;
          __syncthreads();
        } else {
        float acc[9];
#pragma unroll
        for (int q = 0; q < 9; q++) acc[q] = 0.0f;
        for (int base = my0; base < my1; base += 2 * HS_THREADS) {  // two points per thread, their eight cell loads in flight together
          const int ia = base + tid, ib = base + tid + HS_THREADS;
          const int n = my1;  // (shadows the scan length inside the per-point phase: this CTA's share ends at my1)
          float2 pa = make_float2(0.0f, 0.0f), pb = pa;
          HsFetch fa, fb;
          fa.inside = fb.inside = false;
          if (ia < n) { pa = make_float2(__fmul_rn(spts[ia].x, factor), __fmul_rn(spts[ia].y, factor)); fa = hs_point_fetch(prob, m.sx, m.sy, pa, c, s, e0, e1); }
          if (ib < n) { pb = make_float2(__fmul_rn(spts[ib].x, factor), __fmul_rn(spts[ib].y, factor)); fb = hs_point_fetch(prob, m.sx, m.sy, pb, c, s, e0, e1); }
          float ta[9], tb[9];
          if (ia < n) {
            hs_point_terms(fa, pa, sin_rot, cos_rot, ta);
            if (exact) {
#pragma unroll
              for (int q = 0; q < 9; q++) terms[q * pitch + ia] = ta[q];
            } else {
#pragma unroll
              for (int q = 0; q < 9; q++) acc[q] += ta[q];
            }
          }
          if (ib < n) {
            hs_point_terms(fb, pb, sin_rot, cos_rot, tb);
            if (exact) {
#pragma unroll
              for (int q = 0; q < 9; q++) terms[q * pitch + ib] = tb[q];
            } else {
#pragma unroll
              for (int q = 0; q < 9; q++) acc[q] += tb[q];
            }
          }
        }
        if (!exact) {
#pragma unroll
          for (int q = 0; q < 9; q++) {
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], d);
          }
          if (lane == 0) {
#pragma unroll
            for (int q = 0; q < 9; q++) terms[q * NW + warp] = acc[q];
          }
        }
        __syncthreads();
        if (exact) {
          // The reference's float32 sums, in point order (OccGridMapUtil.h:99-126): ONE warp instruction advances all nine
          // chains (lane q owns sum q), so the floor is one dependent FADD per point.  (Nine warps with one chain each
          // share four schedulers and were slower.)
          if (warp == 0 && lane < 9) {
            float acc = 0.0f;
            const float *col = terms + lane * pitch;
            int i = 0;
            for (; i + 32 <= n; i += 32) {  // eight 16-byte loads in flight ahead of the 32 dependent adds they feed
              float4 t[8];
#pragma unroll
              for (int j = 0; j < 8; j++) t[j] = *reinterpret_cast<const float4 *>(col + i + 4 * j);
#pragma unroll
              for (int j = 0; j < 8; j++) {
                acc = __fadd_rn(acc, t[j].x); acc = __fadd_rn(acc, t[j].y); acc = __fadd_rn(acc, t[j].z); acc = __fadd_rn(acc, t[j].w);
              }
            }
            for (; i + 8 <= n; i += 8) {
              const float4 u = *reinterpret_cast<const float4 *>(col + i), w = *reinterpret_cast<const float4 *>(col + i + 4);
              acc = __fadd_rn(acc, u.x); acc = __fadd_rn(acc, u.y); acc = __fadd_rn(acc, u.z); acc = __fadd_rn(acc, u.w);
              acc = __fadd_rn(acc, w.x); acc = __fadd_rn(acc, w.y); acc = __fadd_rn(acc, w.z); acc = __fadd_rn(acc, w.w);
            }
            for (; i < n; i++) acc = __fadd_rn(acc, col[i]);
            tot[lane] = acc;
          }
          __syncthreads();
        } else if (warp == 0) {
          float v = 0.0f;
          if (lane < 9)
            for (int w = 0; w < NW; w++) v += terms[lane * NW + w];
          if (lane < 9) tot[lane] = v;
          __syncwarp();
        }
        }  // !CLUSTER
        if (tid == 0) {  // estimateTransformationLogLh (ScanMatcher.h:107-141)
          const float dTr[3] = {tot[0], tot[1], tot[2]};
          float Hm[9];
          Hm[0] = tot[3]; Hm[4] = tot[4]; Hm[8] = tot[5];
          Hm[1] = Hm[3] = tot[6]; Hm[2] = Hm[6] = tot[7]; Hm[5] = Hm[7] = tot[8];
          float n0 = bc[0], n1 = bc[1], n2 = bc[2];
          if (Hm[0] != 0.0f && Hm[4] != 0.0f) {
            float dir[3];
            inv3_mul(Hm, dTr, dir);
            if (dir[2] > 0.2f) dir[2] = 0.2f;
            else if (dir[2] < -0.2f) dir[2] = -0.2f;
            n0 += dir[0]; n1 += dir[1]; n2 += dir[2];
          }
          bc[0] = n0; bc[1] = n1; bc[2] = n2;
          if (it + 1 < m.iterations) {
            const HsTrig tr = hs_trig(n2, exact, use_fma);
            bc[3] = tr.c; bc[4] = tr.s; bc[5] = tr.sin_rot; bc[6] = tr.cos_rot;
          }
        }
        if (CLUSTER && warp == 0 && it + 1 < m.iterations) {
          __syncwarp();
          publish();
        }
        __syncthreads();
      }
      {
        const float e0 = bc[0], e1 = bc[1], e2 = bc[2];
        const float a = util_normalize_angle(e2);
        get_world_coords(m.tf, e0, e1, world0, world1);
        world2 = a;
        any = true;
      }
      __syncthreads();  // bc / tot are rewritten by the next level
    }
  }
  if (tid == 0) {
    // ---- HectorSlamProcessor::update after the match (:88-107) ----
    float est[3] = {world0, world1, world2};
    if (any) {  // covMatrix = H of the last level matched (level 0)
      lcov[0] = tot[3]; lcov[4] = tot[4]; lcov[8] = tot[5];
      lcov[1] = lcov[3] = tot[6]; lcov[2] = lcov[6] = tot[7];
      lcov[5] = lcov[7] = tot[8];
#pragma unroll
      for (int q = 0; q < 9; q++) st->last_cov[q] = lcov[q];
    }
    const float origo_x = INGEST ? st->origo[0][0] : C.origo_x, origo_y = INGEST ? st->origo[0][1] : C.origo_y;
    if (!C.map_without_matching) {
      st->n_matched = n_matched0 + 1;
      if (n > 0) {
        float factor = 1.0f;
        for (int l = 1; l < Q.levels; l++) {
          factor *= 0.5f;
          st->n_pts[l] = n;
          st->origo[l][0] = origo_x * factor; st->origo[l][1] = origo_y * factor;
        }
      } else {
        for (int l = 1; l < Q.levels; l++) st->n_pts[l] = 0;  // setFrom of an empty container
      }
    }
    st->n_pts[0] = n;
    st->origo[0][0] = origo_x; st->origo[0][1] = origo_y;
    st->last_match_pose[0] = est[0]; st->last_match_pose[1] = est[1]; st->last_match_pose[2] = est[2];
    if (C.carry) { C.carry[0] = est[0]; C.carry[1] = est[1]; C.carry[2] = est[2]; }
    const bool do_update = hs_pose_difference_larger_than(est, lup, Q.min_dist, Q.min_angle) ||
                           C.map_without_matching;
    st->do_update = do_update ? 1 : 0;
    if (do_update) {
      float uc, us;  // Rotation2Df of the update transform: glibc cosf / sinf -> the same cells as the CPU
      glibc_sincosf(est[2], use_fma, &us, &uc);
      for (int l = 0; l < Q.levels; l++) {
        const HsLevel &m = Q.l[l];
        float mx, my;
        get_map_coords(m.tf, est[0], est[1], mx, my);
        st->uc[l] = uc; st->us[l] = us; st->umx[l] = mx; st->umy[l] = my;
        const int2 b0 = begin_cell(uc, us, mx, my, st->origo[l][0], st->origo[l][1]);
        st->bx[l] = b0.x; st->by[l] = b0.y;
        st->epoch[l] += 1;
        st->epoch_hi[l] = st->epoch[l] << 12;
        st->mark_free[l] = st->curr_update_index[l] + 1;  // OccGridMapBase.h:120-121
        st->mark_occ[l] = st->curr_update_index[l] + 2;
        st->curr_update_index[l] += 3;                    // :167
      }
      st->last_update_pose[0] = est[0]; st->last_update_pose[1] = est[1]; st->last_update_pose[2] = est[2];
      st->n_updated += 1;
    }
    float *o = C.out + 16 * (size_t)row;
    o[0] = est[0]; o[1] = est[1]; o[2] = est[2];
    for (int q = 0; q < 9; q++) o[3 + q] = lcov[q];
    o[12] = do_update ? 1.0f : 0.0f;
    o[13] = any ? 1.0f : 0.0f;
    o[14] = (CLUSTER && s_lost) ? 1.0f : 0.0f;  // a cluster exchange timed out: the host fails the call
    if (C.mailbox && b == 0) {
      for (int q = 0; q < 15; q++) C.mailbox[q] = o[q];
      __threadfence_system();
      reinterpret_cast<volatile unsigned int *>(C.mailbox)[15] = C.seq;
      __threadfence_system();
    }
    s_do = do_update ? 1 : 0;
  }
  __syncthreads();
  if (s_do) {
    // cells the rays of this update can touch, per level: the apply pass sweeps this box instead of re-walking the rays
    if (tid < HS_L * 4) s_bb[tid >> 2][tid & 3] = (tid & 2) ? -2147483647 : 2147483647;  // {min x, min y, max x, max y}
    __syncthreads();
    for (int lv = 0; lv < Q.levels; lv++) {
      const HsLevel &m = Q.l[lv];
      const int nl = st->n_pts[lv];
      const float c = st->uc[lv], s = st->us[lv], mx = st->umx[lv], my = st->umy[lv];
      const int bx = st->bx[lv], by = st->by[lv];
      const float2 *pp = reinterpret_cast<const float2 *>(m.pts);
      int lo_x = 2147483647, lo_y = 2147483647, hi_x = -2147483647, hi_y = -2147483647;
      for (int i = tid; i < nl; i += HS_THREADS) {
        const float2 pt = pp[i];
        const BresenhamLine ln = bresenham_line(bx, by, end_cell(c, s, mx, my, pt.x, pt.y), m.sx, m.sy);
        if (!ln.ok) continue;
        lo_x = min(lo_x, min(ln.x0, ln.x1)); hi_x = max(hi_x, max(ln.x0, ln.x1));
        lo_y = min(lo_y, min(ln.y0, ln.y1)); hi_y = max(hi_y, max(ln.y0, ln.y1));
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        lo_x = min(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, d)); lo_y = min(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, d));
        hi_x = max(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, d)); hi_y = max(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, d));
      }
      if (lane == 0) {
        atomicMin(&s_bb[lv][0], lo_x); atomicMin(&s_bb[lv][1], lo_y);
        atomicMax(&s_bb[lv][2], hi_x); atomicMax(&s_bb[lv][3], hi_y);
      }
    }
    __syncthreads();
    if (tid < Q.levels) {
      st->bb_x0[tid] = s_bb[tid][0]; st->bb_y0[tid] = s_bb[tid][1];
      st->bb_x1[tid] = s_bb[tid][2]; st->bb_y1[tid] = s_bb[tid][3];  // no ray: max < min -> an empty box
    }
  }
  if (tid == 0) st->t_match_ns = hs_now_ns() - t0;
  if (CLUSTER) *xc_parity = part_parity;
  const bool verdict = s_do != 0;
  if (C.tag) {
    __syncthreads();  // the bounding boxes (other threads' stores) are ordered before the release below
    if (tid == 0)
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(C.out + 16 * (size_t)row + 15), "r"(C.tag) : "memory");
  }
  return verdict;
}

// every CTA but the matching one: wait until scan i's row carries this launch's tag, then read the gate's verdict
__device__ __forceinline__ bool hs_wait_decision(const float *row, unsigned int tag, int *s_flag) {
  if (threadIdx.x == 0) {
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(row + 15) : "memory");
      if (v == tag) break;
      __nanosleep(40);
    }
    *s_flag = __ldcg(row + 12) != 0.0f ? 1 : 0;
  }
  __syncthreads();
  const bool r = *s_flag != 0;
  __syncthreads();  // s_flag may be rewritten for the next scan
  return r;
}

// A helper CTA of cluster 0 (rank >= 1): the same level / iteration loops as hs_match_cta, but only the per-point phase of
// its share of the scan; the pose comes from the master, the nine partial sums go back to it.
__device__ void hs_match_helper(const HsBatch &P, const HsProc &Q, const HsCall &C, unsigned char *smem, HsXchg *xc, uint32_t rank,
                                uint32_t csize, uint32_t &pose_parity) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = C.n0_uniform;
  if (C.map_without_matching || n <= 0) return;
  float2 *spts = reinterpret_cast<float2 *>(smem);
  float *terms = reinterpret_cast<float *>(smem + hs_terms_offset(P.cap));
  int p0, p1;
  hs_share(n, (int)rank, (int)csize, p0, p1);
  const int cnt = p1 - p0;
  const float2 *gp = reinterpret_cast<const float2 *>(C.pts0);
  for (int i = tid; i < cnt; i += HS_THREADS) spts[i] = gp[p0 + i];
  __syncthreads();
  const int pitch = hs_pitch(P.cap);
  const uint32_t r_part = hs_mapa(smem_u32(&xc->part[rank][0]), 0), r_bar = hs_mapa(smem_u32(&xc->bar_part), 0);
  float factor = 1.0f;
  for (int l = 1; l < Q.levels; l++) factor *= 0.5f;
  for (int lv = Q.levels - 1; lv >= 0; lv--, factor *= 2.0f) {
    const HsLevel &m = Q.l[lv];
    const float4 *prob = m.quad;
    for (int it = 0; it < m.iterations; it++) {
      if (tid == 0) mbar_expect_tx(&xc->bar_pose, 4u * HS_POSE_WORDS);
      mbar_wait_bounded(&xc->bar_pose, pose_parity);  // every thread observes the phase itself (a time-out is reported by the master)
      pose_parity ^= 1u;
      // Not needed for ordering — the master sends this pose only after it holds all nine sums of the previous iteration,
      // which are sent after the column reads — but that chain runs through another CTA, which compute-sanitizer's
      // racecheck cannot follow: the barrier keeps the tool's report clean.
      __syncthreads();
      const float e0 = xc->pose[0], e1 = xc->pose[1], c = xc->pose[3], s = xc->pose[4], sin_rot = xc->pose[5], cos_rot = xc->pose[6];
      const float v = hs_share_sums(prob, m.sx, m.sy, spts, cnt, factor, e0, e1, c, s, sin_rot, cos_rot, terms, pitch, tid, lane, warp);
      if (warp < 9 && lane == 0) hs_st_async(r_part + 4 * warp, v, r_bar);
    }
  }
}

// the update parameters of one level as the gate wrote them.  Plain (L1) loads: within the persistent launch every CTA
// passes the grid barrier between the gate's writes and these reads, and the barrier's gpu-scope acquire drops the SM's
// L1 (CCTL.IVALL); in the batch path a kernel boundary lies in between.  (With L2 loads the ~dozen dependent state reads
// at the head of every warp dominated k_hs_apply's stall samples.)
struct HsUpd {
  int n;
  float c, s, mx, my;
  int bx, by;
  uint32_t ehi;
  int mark_free, mark_occ;
};
__device__ __forceinline__ HsUpd hs_load_upd(const HsState *st, int lv) {
  HsUpd u;
  u.n = st->n_pts[lv];
  u.c = st->uc[lv]; u.s = st->us[lv]; u.mx = st->umx[lv]; u.my = st->umy[lv];
  u.bx = st->bx[lv]; u.by = st->by[lv];
  u.ehi = st->epoch_hi[lv];
  u.mark_free = st->mark_free[lv]; u.mark_occ = st->mark_occ[lv];
  return u;
}

// MapRepMultiMap::updateByScan (:174-191) for processor b, PASS 1 (mark): work item = (level, beam), flattened over
// the levels, one warp each; lanes over Bresenham steps in closed form.  Every traversed cell records the LOWEST beam
// index that frees it / ends on it (32-bit atomicMax of epoch | ~beam).  Returns this warp's cell visits.
__device__ unsigned long long hs_mark_pass(const HsBatch &P, const HsProc &Q, int b, int w, int nw, int lane) {
  const HsState *st = P.state + b;
  unsigned long long my_visits = 0;
  int first[HS_L + 1];
  first[0] = 0;
  for (int lv = 0; lv < Q.levels; lv++) first[lv + 1] = first[lv] + st->n_pts[lv];
  int lv = 0;
  HsUpd u = hs_load_upd(st, 0);
  for (int j = w; j < first[Q.levels]; j += nw) {
    if (j >= first[lv + 1]) {
      while (j >= first[lv + 1]) lv++;
      u = hs_load_upd(st, lv);
    }
    const int i = j - first[lv];
    const HsLevel &m = Q.l[lv];
    uint32_t *fs = m.free_st, *os = m.occ_st;
    const float2 pt = __ldcg(reinterpret_cast<const float2 *>(m.pts) + i);
    const BresenhamLine ln = bresenham_line(u.bx, u.by, end_cell(u.c, u.s, u.mx, u.my, pt.x, pt.y), m.sx, m.sy);
    if (!ln.ok) continue;
    const uint32_t stamp = u.ehi | (uint32_t)(4095 - i);
    const int start = ln.y0 * m.sx + ln.x0;
    for (unsigned int k = lane; k < ln.da; k += 32) atomicMax(fs + bresenham_offset(ln, start, k), stamp);
    if (lane == 0) {
      atomicMax(os + (ln.y1 * m.sx + ln.x1), stamp);
      my_visits += (unsigned long long)ln.da + 1;
    }
  }
  return my_visits;
}

// the probability of cell (x, y) enters the quads of (x, y), (x-1, y), (x, y-1), (x-1, y-1)
__device__ __forceinline__ void hs_publish_prob(float4 *__restrict__ quad, int sx, int x, int y, float p) {
  float *q = reinterpret_cast<float *>(quad + (y * sx + x));
  q[0] = p;
  if (x > 0) q[-4 + 1] = p;
  if (y > 0) {
    q[-4 * sx + 2] = p;
    if (x > 0) q[-4 * sx - 4 + 3] = p;
  }
}

// PASS 2 (apply): a dense, coalesced sweep over each level's bounding box of the rays (work item = 128 consecutive
// cells of a row: four 128-byte loads per stamp plane per warp).  A cell stamped in this epoch gets the reference's
// update exactly once: end cells (occ stamp of this epoch; the stamp's winner is the lowest beam ending there) take
// bresenhamCellOcc — with the "(v + f) - f" un-free rounding iff a LOWER beam index had freed the cell first (its
// free stamp, same epoch, is larger) — then += logOddsOccupied if v < 50; cells only freed take bresenhamCellFree.
// The floats are those of the sequential loop (OccGridMapBase.h:302-330), whatever the execution order.
__device__ void hs_apply_pass(const HsBatch &P, const HsProc &Q, int b, int w, int nw, int lane) {
  const HsState *st = P.state + b;
  int first[HS_L + 1], x0[HS_L], y0[HS_L], x1[HS_L], chunks[HS_L];
  first[0] = 0;
  for (int lv = 0; lv < Q.levels; lv++) {
    x0[lv] = st->bb_x0[lv]; y0[lv] = st->bb_y0[lv];
    x1[lv] = st->bb_x1[lv];
    const int y1 = st->bb_y1[lv];
    const bool any = x1[lv] >= x0[lv] && y1 >= y0[lv];
    chunks[lv] = any ? (x1[lv] - x0[lv] + 128) / 128 : 0;
    first[lv + 1] = first[lv] + (any ? (y1 - y0[lv] + 1) * chunks[lv] : 0);
  }
  int lv = 0;
  for (int j = w; j < first[Q.levels]; j += nw) {
    while (j >= first[lv + 1]) lv++;
    const HsLevel &m = Q.l[lv];
    const uint32_t *fs = m.free_st, *os = m.occ_st;
    float *lo = m.lo;
    float4 *quad = m.quad;
    int32_t *ui = m.ui;
    const uint32_t ep = st->epoch_hi[lv] >> 12;
    const int mark_free = st->mark_free[lv], mark_occ = st->mark_occ[lv];
    const int r = j - first[lv];
    const int y = y0[lv] + r / chunks[lv];
    const int xb = x0[lv] + (r % chunks[lv]) * 128 + lane;
    uint32_t f[4], o[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int x = xb + 32 * q;
      f[q] = o[q] = 0;
      if (x <= x1[lv]) {
        f[q] = __ldcg(fs + (y * m.sx + x));
        o[q] = __ldcg(os + (y * m.sx + x));
      }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int off = y * m.sx + xb + 32 * q;
      if (o[q] != 0 && (o[q] >> 12) == ep) {  // bresenhamCellOcc (:315-330)
        float v = __ldcg(lo + off);
        if ((f[q] >> 12) == ep && f[q] > o[q]) {  // a lower beam index freed it first: set free, then unset
          v = __fadd_rn(v, Q.lo_free);
          v = __fsub_rn(v, Q.lo_free);
        }
        if (v < 50.0f) v = __fadd_rn(v, Q.lo_occ);
        lo[off] = v;
        hs_publish_prob(quad, m.sx, xb + 32 * q, y, log_odds_prob(v));
        ui[off] = mark_occ;
      } else if (f[q] != 0 && (f[q] >> 12) == ep) {  // bresenhamCellFree (:302-312)
        const float v = __fadd_rn(__ldcg(lo + off), Q.lo_free);
        lo[off] = v;
        hs_publish_prob(quad, m.sx, xb + 32 * q, y, log_odds_prob(v));
        ui[off] = mark_free;
      }
    }
  }
}

// ---- batch path: three launches per step over all B processors ----
// The match kernels run one CTA per SM.  Their launch bounds say so: without the minimum of one block, ptxas may cap
// the registers at 56 to fit two 576-thread CTAs on an SM, and spills.
template <bool EXACT>
__global__ void __launch_bounds__(HS_THREADS, 1) k_hs_match(HsBatch P, HsCall C) {
  extern __shared__ __align__(16) unsigned char hs_smem[];
  __shared__ HsProc s_proc;
  hs_load_proc(P, blockIdx.x, &s_proc);
  hs_match_cta<EXACT, false>(P, s_proc, C, blockIdx.x, hs_smem);
}
// processors b = blockIdx.y, + gridDim.y, ... (grid_rows(batch) rows)
__global__ void __launch_bounds__(256) k_hs_mark(HsBatch P) {
  __shared__ HsProc s_proc;
  for (int b = blockIdx.y; b < P.batch; b += gridDim.y) {
    if (!P.state[b].do_update) continue;
    hs_load_proc(P, b, &s_proc);
    const int lane = threadIdx.x & 31;
    const unsigned long long v = hs_mark_pass(P, s_proc, b, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, (gridDim.x * blockDim.x) >> 5, lane);
    if (lane == 0 && v) atomicAdd(&P.state[b].visits, v);  // lane 0 carries the warp's count
    __syncthreads();  // s_proc is rewritten for the next processor
  }
}
__global__ void __launch_bounds__(256) k_hs_apply(HsBatch P) {
  __shared__ HsProc s_proc;
  for (int b = blockIdx.y; b < P.batch; b += gridDim.y) {
    if (!P.state[b].do_update) continue;
    hs_load_proc(P, b, &s_proc);
    hs_apply_pass(P, s_proc, b, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, (gridDim.x * blockDim.x) >> 5, threadIdx.x & 31);
    __syncthreads();
  }
}

// ---- single-processor path: ONE cooperative launch walks n_scans scans (n_scans = 1 for b2s_hector_slam_update) ----
// CTA 0 matches while the other CTAs wait at the grid barrier; then every CTA takes beams of the update passes.
__device__ __forceinline__ void hs_grid_barrier(unsigned int *counter, unsigned int &generation) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int target = (generation + 1) * gridDim.x;
    atomicAdd(counter, 1u);
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v >= target) break;
      __nanosleep(40);
    }
    __threadfence();
  }
  generation++;
  __syncthreads();
}

struct HsStream {
  const float *pts;      // concatenated scans (device, or host-mapped for a single scan)
  const int *offsets;    // [n_scans] first point of each scan, or NULL (single scan at 0)
  const int *counts;     // [n_scans] or NULL -> count0
  int count0, n_scans;
  const float *hints;    // [n_scans][3] or NULL (chain through the processor's last scan-match pose)
  const float *first_hint;  // device [3] or NULL
  float origo_x, origo_y;
  int map_without_matching;
  float *out;            // [n_scans][16]
  volatile float *mailbox;
  unsigned int seq;
  unsigned int *barrier;
  unsigned int tag;      // this launch's id (never 0): scan i is decided once out[i][15] holds it
};

template <bool EXACT, bool CLUSTER>
__global__ void __launch_bounds__(HS_THREADS, 1) k_hs_stream(HsBatch P, HsStream S) {
  extern __shared__ __align__(16) unsigned char hs_smem[];
  __shared__ HsXchg xc;  // same offset in every CTA of the kernel: mapa() of a local address names the peer's copy
  __shared__ int s_flag;
  __shared__ HsProc s_proc;
  hs_load_proc(P, 0, &s_proc);
  uint32_t crank = 0, csize = 1, pose_parity = 0, part_parity = 0;
  if (CLUSTER) {
    crank = hs_cluster_rank();
    csize = hs_cluster_size();
    if (threadIdx.x == 0) {
      mbar_init(&xc.bar_pose, 1);
      mbar_init(&xc.bar_part, 1);
      fence_mbar_init();
    }
    hs_cluster_sync();  // no peer signals a barrier that is not initialised yet (once per launch)
  }
  const bool helper = CLUSTER && blockIdx.x < csize && crank != 0;  // cluster 0 = CTAs [0, csize)
  unsigned int generation = 0;
  const int lane = threadIdx.x & 31;
  const int w = (blockIdx.x * HS_THREADS + threadIdx.x) >> 5, nw = (gridDim.x * HS_THREADS) >> 5;
  HsState *st = P.state;
  __shared__ float s_last[3];  // the matching CTA's last scan-match pose: the next scan's hint without a global round trip
  int next_off = (S.offsets && S.n_scans > 0) ? S.offsets[0] : 0, next_cnt = (S.counts && S.n_scans > 0) ? S.counts[0] : S.count0;
  for (int i = 0; i < S.n_scans; i++) {
    bool update;
    HsCall C;
    const int off = next_off, cnt_i = next_cnt;
    if (i + 1 < S.n_scans) {  // requested a whole scan ahead of their use
      if (S.offsets) next_off = S.offsets[i + 1];
      if (S.counts) next_cnt = S.counts[i + 1];
    }
    C.pts0 = S.pts + 2 * (size_t)off;
    C.n0 = nullptr;
    C.n0_uniform = cnt_i;
    C.pts_stride = 0;
    C.hints = S.hints ? S.hints + 3 * (size_t)i : ((i == 0 && S.first_hint) ? S.first_hint : (i > 0 ? s_last : nullptr));
    C.carry = s_last;
    C.origo_x = S.origo_x; C.origo_y = S.origo_y;
    C.map_without_matching = S.map_without_matching;
    C.out = S.out + 16 * (size_t)i;
    C.mailbox = S.mailbox;
    C.seq = S.seq;
    C.tag = S.tag;
    // The matching CTA never waits for the others unless the map is updated: it publishes the scan's verdict (release) and
    // goes on to the next scan; the other CTAs follow the verdicts and meet it at the update's barriers.  (A grid barrier
    // per scan cost the matching CTA ~1 us: two fences and an L2 round trip.)
    if (blockIdx.x == 0) {
      update = hs_match_cta<EXACT, CLUSTER>(P, s_proc, C, 0, hs_smem, &xc, &part_parity);
    } else {
      if (helper) hs_match_helper(P, s_proc, C, hs_smem, &xc, crank, csize, pose_parity);
      update = hs_wait_decision(C.out, S.tag, &s_flag);
    }
    if (update) {
      const unsigned long long t0 = hs_now_ns();
      const unsigned long long v = hs_mark_pass(P, s_proc, 0, w, nw, lane);
      if (lane == 0 && v) atomicAdd(&st->visits, v);
      hs_grid_barrier(S.barrier, generation);
      hs_apply_pass(P, s_proc, 0, w, nw, lane);
      hs_grid_barrier(S.barrier, generation);  // the next match reads the refreshed probability planes
      if (blockIdx.x == 0 && threadIdx.x == 0) st->t_update_ns = hs_now_ns() - t0;
    }
  }
}

// ---- batched streams: ONE launch, one CTA per processor, each walking its own recording ----
struct HsFleet {
  const float *pts;          // every scan's points, processor-major ([sum n_points][2])
  const long long *offsets;  // [total scans] first point of each scan (64-bit: a fleet's recordings exceed 2^31 floats)
  const int *counts;         // [total scans]
  const long long *first;    // [B][2] processor b's scans first[2b] ... first[2b + 1] - 1 (a node call's part ends a
                             // processor's scans before the next one's begin)
  const float *hints;        // [total scans][3] or NULL (chain through the processor's last scan-match pose)
  const float *first_hints;  // [B][3] or NULL: hint of each processor's first scan when chaining
  float origo_x, origo_y;    // (ingest: unused, each processor's own is in its state)
  int map_without_matching;
  float *out;                // [total scans][16]
  const struct HsIngest *ingest;  // device: the ingest kernel's input (k_hs_stream_batch<_, true>), else NULL
};

// Scans as raw LaserScan ranges (k_hs_stream_batch<_, true>): F.pts / offsets / counts are unused.  In device memory
// behind one pointer: a larger kernel parameter block costs the point-stream instantiations registers.
struct HsIngest {
  const float *ranges;       // every scan's ranges, float32 (HsLaser::base)
  const double2 *units;      // the beams' unit vectors (host C library cos / sin), per laser (HsLaser::unit0)
  const HsLaser *lasers;     // [B]
};

// The loop of processor b = blockIdx.x over its scans: match (hs_match_cta), then, if the gate opens, the mark and
// apply passes on this CTA's 18 warps.  Nothing crosses CTAs: no grid barrier, no verdict tags, and B may exceed the
// resident CTAs (later processors start as earlier ones finish).  The match reads the probability quads with plain
// (L1-allocating, coherent) loads that the SAME CTA rewrote in its previous apply pass; the __syncthreads after the
// apply orders those stores before the loads (CTA scope), so no L1 drop is needed as in k_hs_stream.
//
// INGEST: each scan arrives as n_ranges float32 ranges.  Before its match the CTA converts it with processor b's filter
// (hector_scan.cuh: the node's projectLaser + rosPointCloudToDataContainer, per beam) and compacts the kept beams in
// beam order into its level-0 container row, HS_THREADS beams per round: ballot / popc inside a warp, warp offsets
// through shared memory, a running base across rounds.  hs_match_cta then reads that row as its input and copies it
// onto itself: each element is read and written back unchanged by the same thread, which is benign.  The container's
// origo is the processor's own (hs_match_cta<_, _, true>).
template <bool EXACT, bool INGEST>
__global__ void __launch_bounds__(HS_THREADS, 1) k_hs_stream_batch(HsBatch P, HsFleet F) {
  extern __shared__ __align__(16) unsigned char hs_smem[];
  __shared__ float s_last[3];  // the previous scan's match pose: the next scan's hint without a global round trip
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = HS_THREADS / 32;
  HsState *st = P.state + b;
  __shared__ HsProc s_proc;
  hs_load_proc(P, b, &s_proc);
  const long long s0 = F.first[2 * b], s1 = F.first[2 * b + 1];
  unsigned long long visits = 0;
  for (long long i = s0; i < s1; i++) {
    HsCall C;
    if constexpr (INGEST) {
      __shared__ int s_warp_kept[NW];
      const HsIngest &I = *F.ingest;
      const HsLaser &las = I.lasers[b];
      float2 *row = reinterpret_cast<float2 *>(s_proc.l[0].pts);
      const int nr = las.n_ranges;
      const float *r = I.ranges + (las.base + i * nr);
      const double2 *units = I.units + las.unit0;
      int base = 0;
      for (int c0 = 0; c0 < nr; c0 += HS_THREADS) {
        const int j = c0 + (int)threadIdx.x;
        float2 q = make_float2(0.0f, 0.0f);
        bool keep = false;
        if (j < nr) {
          const double2 u = units[j];
          keep = hector_node_beam(las.filter, r[j], u.x, u.y, las.range_cutoff, las.range_min, q.x, q.y);
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp_kept[warp] = __popc(m);
        __syncthreads();
        int off = base, round = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) {
          const int k = s_warp_kept[w];
          off += w < warp ? k : 0;
          round += k;
        }
        if (keep) row[off + __popc(m & ((1u << lane) - 1u))] = q;
        base += round;
        __syncthreads();  // s_warp_kept is rewritten by the next round; the row is read by the match
      }
      if (threadIdx.x == 0) F.out[16 * i + 15] = __int_as_float(base);  // the scan's kept-beam count for the host
      C.pts0 = s_proc.l[0].pts;
      C.n0 = nullptr;
      C.n0_uniform = base;
    } else {
      C.pts0 = F.pts + 2 * F.offsets[i];
      C.n0 = nullptr;
      C.n0_uniform = F.counts[i];
    }
    C.pts_stride = 0;
    C.hints = F.hints ? F.hints + 3 * i : (i > s0 ? s_last : (F.first_hints ? F.first_hints + 3 * (size_t)b : nullptr));
    C.origo_x = F.origo_x; C.origo_y = F.origo_y;
    C.map_without_matching = F.map_without_matching;
    C.out = F.out + 16 * i;
    C.mailbox = nullptr;
    C.seq = 0;
    C.tag = 0;
    C.carry = s_last;
    C.own_row = 1;
    if (hs_match_cta<EXACT, false, INGEST>(P, s_proc, C, b, hs_smem)) {
      const unsigned long long t0 = hs_now_ns();
      visits += hs_mark_pass(P, s_proc, b, warp, NW, lane);  // (lane 0 carries the warp's count)
      __syncthreads();
      hs_apply_pass(P, s_proc, b, warp, NW, lane);
      __syncthreads();  // the next match reads the refreshed quads; the next gate rewrites the update parameters
      if (threadIdx.x == 0) st->t_update_ns = hs_now_ns() - t0;
    }
  }
  if (lane == 0 && visits) atomicAdd(&st->visits, visits);
}

__global__ void k_hs_fill(float *__restrict__ p, size_t n, float v) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void k_hs_state_init(HsState *st, int batch, int reset_maps) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  HsState &s = st[b];
  // HectorSlamProcessor::reset (:111-116)
  s.last_update_pose[0] = s.last_update_pose[1] = s.last_update_pose[2] = 3.402823466e+38F;
  s.last_match_pose[0] = s.last_match_pose[1] = s.last_match_pose[2] = 0.0f;
  s.do_update = 0;
  if (reset_maps == 2) {  // create
    for (int q = 0; q < 9; q++) s.last_cov[q] = 0.0f;
    for (int l = 0; l < HS_L; l++) { s.curr_update_index[l] = 0; s.epoch[l] = 0; s.n_pts[l] = 0; s.origo[l][0] = s.origo[l][1] = 0.0f; }
    s.visits = s.n_matched = s.n_updated = 0;
    s.t_match_ns = s.t_update_ns = 0;
    for (int l = 0; l < HS_L; l++) { s.bb_x0[l] = s.bb_y0[l] = 0; s.bb_x1[l] = s.bb_y1[l] = -1; }
  }
}

__global__ void k_hs_epoch_reset(HsState *st, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  for (int l = 0; l < HS_L; l++) st[b].epoch[l] = 0;
}

}  // namespace b2s

struct b2s_hector_slam {
  Stream stream;
  int device = 0;
  int levels = 0;  // the most levels of any processor
  int batch = 1, cap = 0;
  std::vector<b2s_hector_map_spec> specs;  // [batch]
  std::vector<HsProc> procs;               // [batch] the host copy of the device table P.procs
  Buf<HsProc> d_procs;
  HsBatch P;
  struct {  // level l's pools: the planes of every processor with more than l levels, back to back
    Buf<float4> quad;
    Buf<float> lo, pts;
    Buf<int32_t> ui;
    Buf<uint32_t> free_st, occ_st;
    size_t cells = 0;
  } level_mem[HS_L];
  Buf<HsState> d_state;
  Buf<float> d_out;                // [batch][16] (per-scan / batch calls)
  HostBuf<float> h_out;            // pinned [batch][16]
  HostBuf<float> h_pts;            // host-mapped pinned staging of one scan (single-processor call)
  HostBuf<volatile float> h_mail;  // host-mapped mailbox [16]
  HostBuf<float> h_hint;           // host-mapped [3] pose hint of the per-scan call
  unsigned int seq = 0;
  Buf<unsigned int> d_barrier;
  unsigned long long host_updates = 0;  // upper bound of every level's device epoch
  int stream_ctas = HS_STREAM_CTAS;
  bool coop = true;
  unsigned int launch_tag = 0;  // id of the last stream launch (the kernel publishes per-scan verdicts under it)
  int cluster = 1;  // CTAs per thread-block cluster of the fast-mode stream kernel (1: no cluster launch)
  Event ev_done;
  bool launch_pending = false;  // a per-scan launch may still be running its update passes
};

extern "C" void b2s_hector_slam_destroy(b2s_hector_slam *p);

static b2s_status hs_clear_maps(b2s_hector_slam *p) {  // GridMapBase::reset -> clear(): resetGridCell on every cell (:93-113)
  for (int l = 0; l < p->levels; l++) {
    const auto &m = p->level_mem[l];
    const size_t cells = m.cells;
    B2S_CUDA_CHECK(cudaMemsetAsync(m.lo, 0, cells * 4, p->stream));       // logOdds 0
    B2S_CUDA_CHECK(cudaMemsetAsync(m.ui, 0xff, cells * 4, p->stream));    // updateIndex -1
    B2S_CUDA_CHECK(cudaMemsetAsync(m.free_st, 0, cells * 4, p->stream));
    B2S_CUDA_CHECK(cudaMemsetAsync(m.occ_st, 0, cells * 4, p->stream));
    k_hs_fill<<<ceil_div((long long)cells * 4, 256), 256, 0, p->stream>>>(reinterpret_cast<float *>(m.quad.p), cells * 4, 0.5f);  // e^0 / (e^0 + 1)
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  return B2S_OK;
}

// stamps carry a 20-bit epoch: before any level's epoch could overflow, clear the stamps and restart the epochs.
// host_updates counts calls (>= every device epoch), so the test needs no device read-back.
static b2s_status hs_reserve_epochs(b2s_hector_slam *p, unsigned long long n_updates) {
  if (p->host_updates + n_updates < HS_EPOCH_MAX) {
    p->host_updates += n_updates;
    return B2S_OK;
  }
  if (n_updates >= HS_EPOCH_MAX) B2S_FAIL(B2S_ERR_TOO_LARGE, "too many scans in one call (stamp epochs are 20 bits)");
  for (int l = 0; l < p->levels; l++) {
    const auto &m = p->level_mem[l];
    B2S_CUDA_CHECK(cudaMemsetAsync(m.free_st, 0, m.cells * 4, p->stream));
    B2S_CUDA_CHECK(cudaMemsetAsync(m.occ_st, 0, m.cells * 4, p->stream));
  }
  k_hs_epoch_reset<<<ceil_div(p->batch, 128), 128, 0, p->stream>>>(p->d_state, p->batch);
  B2S_CUDA_CHECK(cudaGetLastError());
  p->host_updates = n_updates;
  return B2S_OK;
}

// the handle's table (p->procs) -> the device, in stream order: the next launch on the stream reads it
static b2s_status hs_upload_procs(b2s_hector_slam *p) {
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  B2S_CUDA_CHECK(cudaMemcpyAsync(p->d_procs, p->procs.data(), sizeof(HsProc) * p->procs.size(), cudaMemcpyHostToDevice,
                                 p->stream));  // (pageable source: staged before the call returns)
  return B2S_OK;
}

namespace b2s {

// why HectorSlamProcessor's constructor arguments in `s` are refused, or NULL (the checks of b2s_hector_slam_create):
// levels 1 ... 8, a positive resolution, and more than 2 cells each way on the coarsest level
const char *hs_spec_error(const b2s_hector_map_spec &s) {
  if (s.levels < 1 || s.levels > B2S_HECTOR_MAX_LEVELS) return "levels must be 1 ... 8";
  if (!(s.map_resolution > 0.0f)) return "map_resolution must be positive";
  if ((s.map_size_x >> (s.levels - 1)) <= 2 || (s.map_size_y >> (s.levels - 1)) <= 2)
    return "the map size leaves 2 cells or fewer on the coarsest level";
  return nullptr;
}

// b2s_hector_slam_create's processor with the constructor's update factors and map-update gate
b2s_hector_map_spec hs_default_spec(float map_resolution, int map_size_x, int map_size_y, float start_x, float start_y,
                                    int levels) {
  b2s_hector_map_spec s;
  std::memset(&s, 0, sizeof(s));
  s.map_resolution = map_resolution;
  s.map_size_x = map_size_x; s.map_size_y = map_size_y;
  s.start_x = start_x; s.start_y = start_y;
  s.levels = levels;
  s.update_free = 0.4f; s.update_occupied = 0.6f;  // GridMapLogOdds.h:98-102
  s.min_dist = 0.4f; s.min_angle = 0.13f;          // HectorSlamProcessor.h:63-64
  return s;
}

}  // namespace b2s

// cell length of a processor's level: the resolution doubled per level (MapRepMultiMap.h:56-89)
static float hs_cell_length(const b2s_hector_map_spec &s, int level) {
  float res = s.map_resolution;
  for (int l = 0; l < level; l++) res *= 2.0f;
  return res;
}

// Every spec is checked before the device is touched; `who` names the entry point in refusals.
static b2s_status hs_create(int batch, int max_points, const b2s_hector_map_spec *specs, int device, void *cuda_stream,
                            b2s_hector_slam **out, const char *who) {
  if (!out || !specs || batch < 1 || max_points < 1)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(who) + ": null argument or bad batch / max_points");
  *out = nullptr;
  for (int b = 0; b < batch; b++)
    if (const char *e = hs_spec_error(specs[b]))
      B2S_FAIL(B2S_ERR_BAD_PARAMS, std::string(who) + ": processor " + std::to_string(b) + ": " + e);
  if (max_points > HS_MAX_PTS) B2S_FAIL(B2S_ERR_TOO_LARGE, "at most 4096 points per scan");
  if (b2s_status st = open_device(device)) return st;
  std::unique_ptr<b2s_hector_slam, decltype(&b2s_hector_slam_destroy)> p(new (std::nothrow) b2s_hector_slam(), b2s_hector_slam_destroy);
  if (!p) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  p->device = device;
  p->batch = batch;
  p->cap = max_points;
  p->specs.assign(specs, specs + batch);
  for (int b = 0; b < batch; b++) p->levels = std::max(p->levels, (int)specs[b].levels);
  B2S_CUDA_CHECK(p->stream.init(cuda_stream));
  std::memset(&p->P, 0, sizeof(p->P));
  p->P.batch = batch; p->P.cap = max_points;
  p->P.exact = 1;
  const int variant = glibc_sincosf_variant_of_host();
  p->P.use_fma = variant == 0 ? 0 : 1;
  // the pools: level l holds processor b's planes (b ascending) when b has more than l levels
  std::vector<size_t> at((size_t)batch * HS_L, 0);  // [b][l] processor b's first cell in level l's pool
  for (int l = 0; l < p->levels; l++) {
    size_t cells = 0, rows = 0;
    for (int b = 0; b < batch; b++) {
      if (specs[b].levels <= l) continue;
      at[(size_t)b * HS_L + l] = cells;
      cells += (size_t)(specs[b].map_size_x >> l) * (size_t)(specs[b].map_size_y >> l);
      rows++;
    }
    auto &mem = p->level_mem[l];
    mem.cells = cells;
    B2S_CUDA_CHECK(mem.lo.reserve(cells));
    B2S_CUDA_CHECK(mem.ui.reserve(cells));
    B2S_CUDA_CHECK(mem.free_st.reserve(cells));
    B2S_CUDA_CHECK(mem.occ_st.reserve(cells));
    B2S_CUDA_CHECK(mem.quad.reserve(cells));
    B2S_CUDA_CHECK(mem.pts.reserve(2 * (size_t)max_points * rows));
  }
  p->procs.resize((size_t)batch);
  size_t rows[HS_L] = {};  // container rows handed out so far, per level
  for (int b = 0; b < batch; b++) {
    const b2s_hector_map_spec &s = specs[b];
    HsProc &q = p->procs[(size_t)b];
    std::memset(&q, 0, sizeof(q));
    q.levels = s.levels;
    q.lo_free = prob_to_log_odds(s.update_free);
    q.lo_occ = prob_to_log_odds(s.update_occupied);
    q.min_dist = s.min_dist; q.min_angle = s.min_angle;
    // MapRepMultiMap ctor (MapRepMultiMap.h:56-89): one offset for every level, dims halve, cell length doubles
    const float total_x = s.map_resolution * static_cast<float>(s.map_size_x), total_y = s.map_resolution * static_cast<float>(s.map_size_y);
    const float off_x = total_x * s.start_x, off_y = total_y * s.start_y;
    for (int l = 0; l < s.levels; l++) {
      const size_t row = rows[l]++;
      HsLevel &m = q.l[l];
      m.sx = s.map_size_x >> l; m.sy = s.map_size_y >> l;
      m.tf = map_transform(hs_cell_length(s, l), off_x, off_y);
      m.iterations = 1 + (l == 0 ? 5 : 3);
      const auto &mem = p->level_mem[l];
      const size_t c0 = at[(size_t)b * HS_L + l];
      m.lo = mem.lo.p + c0; m.ui = mem.ui.p + c0; m.free_st = mem.free_st.p + c0; m.occ_st = mem.occ_st.p + c0;
      m.quad = mem.quad.p + c0;
      m.pts = mem.pts.p + 2 * (size_t)max_points * row;
    }
  }
  B2S_CUDA_CHECK(p->d_procs.reserve((size_t)batch));
  p->P.procs = p->d_procs;
  if (b2s_status st = hs_upload_procs(p.get())) return st;
  B2S_CUDA_CHECK(p->d_state.reserve(batch));
  p->P.state = p->d_state;
  B2S_CUDA_CHECK(p->d_out.reserve(16 * (size_t)batch));
  B2S_CUDA_CHECK(p->d_barrier.reserve(1));
  B2S_CUDA_CHECK(p->h_out.reserve(16 * (size_t)batch));
  B2S_CUDA_CHECK(p->h_pts.reserve(2 * (size_t)max_points, cudaHostAllocMapped));
  B2S_CUDA_CHECK(p->h_mail.reserve(16, cudaHostAllocMapped));
  std::memset((void *)p->h_mail.p, 0, sizeof(float) * 16);
  B2S_CUDA_CHECK(p->h_hint.reserve(4, cudaHostAllocMapped));
  B2S_CUDA_CHECK(p->ev_done.create(cudaEventDisableTiming));
  const size_t smem = hs_smem_bytes(max_points);
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_match<true>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_match<false>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream<true, false>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream<false, false>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream<false, true>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream_batch<true, false>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream_batch<false, false>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream_batch<true, true>, smem));
  B2S_CUDA_CHECK(raise_dyn_smem(k_hs_stream_batch<false, true>, smem));
  {
    int coop = 0, sms = 0, per_sm = 0;
    B2S_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    B2S_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    B2S_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_hs_stream<true, false>, HS_THREADS, smem));
    p->coop = coop != 0;
    p->stream_ctas = std::max(1, std::min(HS_STREAM_CTAS, sms * std::max(per_sm, 0)));
    if (!p->coop) p->stream_ctas = 1;  // without a co-residency guarantee a spinning grid barrier could deadlock
    // fast mode: the matching CTA's cluster.  Needs the whole cooperative grid co-resident AS clusters.
    // B2S_HS_CLUSTER=0 keeps the one-CTA match, the path of devices and drivers that cannot do that, so that it can be
    // compared with the cluster match on one that can.
    const char *e = getenv("B2S_HS_CLUSTER");
    if (p->coop && p->stream_ctas >= HS_CLUSTER && !(e && e[0] == '0')) {
      cudaLaunchConfig_t cfg;
      std::memset(&cfg, 0, sizeof(cfg));
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = (unsigned)HS_CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.gridDim = dim3((p->stream_ctas / HS_CLUSTER) * HS_CLUSTER);
      cfg.blockDim = dim3(HS_THREADS);
      cfg.dynamicSmemBytes = smem;
      cfg.attrs = at; cfg.numAttrs = 1;
      int n_clusters = 0;
      if (cudaOccupancyMaxActiveClusters(&n_clusters, k_hs_stream<false, true>, &cfg) == cudaSuccess &&
          n_clusters * HS_CLUSTER >= (int)cfg.gridDim.x)
        p->cluster = HS_CLUSTER;
      else
        cudaGetLastError();
    }
  }
  k_hs_state_init<<<ceil_div(batch, 128), 128, 0, p->stream>>>(p->d_state, batch, 2);
  if (b2s_status st = hs_clear_maps(p.get())) return st;
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  *out = p.release();
  return B2S_OK;
}

// wait until the previous per-scan launch (its update passes) has left the host-mapped staging buffers alone
static b2s_status hs_wait_launch(b2s_hector_slam *p) {
  if (p->launch_pending) {
    B2S_CUDA_CHECK(cudaEventSynchronize(p->ev_done));
    p->launch_pending = false;
  }
  return B2S_OK;
}

static b2s_status hs_launch_stream(b2s_hector_slam *p, const HsStream &S) {
  B2S_CUDA_CHECK(cudaMemsetAsync(p->d_barrier, 0, sizeof(unsigned int), p->stream));
  HsBatch P = p->P;
  HsStream Sv = S;
  Sv.barrier = p->d_barrier;
  p->launch_tag += 1;
  if (p->launch_tag == 0) p->launch_tag = 1;
  Sv.tag = p->launch_tag;
  const size_t smem = hs_smem_bytes(p->cap);
  if (p->coop && !P.exact && p->cluster > 1) {
    // cooperative (all CTAs co-resident for the grid barrier) AND clustered (CTAs [0, cluster) share the match)
    cudaLaunchConfig_t cfg;
    std::memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
    at[1].id = cudaLaunchAttributeClusterDimension;
    at[1].val.clusterDim.x = (unsigned)p->cluster; at[1].val.clusterDim.y = 1; at[1].val.clusterDim.z = 1;
    cfg.gridDim = dim3((p->stream_ctas / p->cluster) * p->cluster);
    cfg.blockDim = dim3(HS_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = p->stream;
    cfg.attrs = at; cfg.numAttrs = 2;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, k_hs_stream<false, true>, P, Sv);
    if (e == cudaSuccess) return B2S_OK;
    cudaGetLastError();
    p->cluster = 1;  // this driver refuses the combination: the one-CTA match from now on
  }
  if (p->coop) {
    void *args[2] = {&P, &Sv};
    const void *kern = P.exact ? reinterpret_cast<const void *>(k_hs_stream<true, false>) : reinterpret_cast<const void *>(k_hs_stream<false, false>);
    B2S_CUDA_CHECK(cudaLaunchCooperativeKernel(kern, dim3(p->stream_ctas), dim3(HS_THREADS), args, smem, p->stream));
  } else {
    if (P.exact) k_hs_stream<true, false><<<1, HS_THREADS, smem, p->stream>>>(P, Sv);
    else k_hs_stream<false, false><<<1, HS_THREADS, smem, p->stream>>>(P, Sv);
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  return B2S_OK;
}

// Processor b's scans of a batched call are first[2b] ... first[2b + 1] - 1 (HsFleet::first), in processor order, so
// the call has first.back() scans.  Refuses negative counts; `longest` is the most scans of one processor.
static b2s_status hs_fleet_counts(const b2s_hector_slam *p, const int32_t *n_scans, std::vector<long long> &first, int &longest) {
  const int B = p->batch;
  first.assign(2 * (size_t)B, 0);
  long long total = 0;
  longest = 0;
  for (int b = 0; b < B; b++) {
    if (n_scans[b] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "negative scan count");
    first[2 * (size_t)b] = total;
    total += n_scans[b];
    first[2 * (size_t)b + 1] = total;
    longest = std::max(longest, (int)n_scans[b]);
  }
  return B2S_OK;
}

// The body the batched stream calls share, once the caller has checked its inputs: hint uploads, ONE k_hs_stream_batch
// launch and the read-back.  `upload(F)` enqueues the scans (points, or raw ranges for INGEST) and fills F's input fields.
template <class Upload>
static b2s_status hs_fleet_run(b2s_hector_slam *p, const int32_t *n_scans, const std::vector<long long> &first, int longest,
                               bool ingest, const float *first_pose_hints, const float *pose_hints, int map_without_matching,
                               float *out_poses, int32_t *out_map_updated, float *out_last_covs, int32_t *out_n_points,
                               Upload &upload) {
  const int B = p->batch;
  const size_t T = (size_t)first.back();
  if (T == 0) return B2S_OK;
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  if ((st = hs_reserve_epochs(p, (unsigned long long)longest))) return st;  // a processor's epochs advance once per scan at most
  HsFleet F;
  std::memset(&F, 0, sizeof(F));
  if ((st = upload(F))) return st;
  AsyncBuf<float> d_hints(p->stream), d_first_hints(p->stream), d_out(p->stream);
  AsyncBuf<long long> d_first(p->stream);
  B2S_CUDA_CHECK(d_first.alloc(first.size()));
  B2S_CUDA_CHECK(d_out.alloc(16 * T));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_first, first.data(), sizeof(long long) * first.size(), cudaMemcpyHostToDevice, p->stream));
  if (pose_hints) {
    B2S_CUDA_CHECK(d_hints.alloc(3 * T));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_hints, pose_hints, sizeof(float) * 3 * T, cudaMemcpyHostToDevice, p->stream));
  } else if (first_pose_hints) {
    B2S_CUDA_CHECK(d_first_hints.alloc(3 * (size_t)B));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_first_hints, first_pose_hints, sizeof(float) * 3 * (size_t)B, cudaMemcpyHostToDevice, p->stream));
  }
  F.first = d_first;
  F.hints = d_hints; F.first_hints = d_first_hints;
  F.map_without_matching = map_without_matching;
  F.out = d_out;
  const size_t smem = hs_smem_bytes(p->cap);
  if (ingest) {
    if (p->P.exact) k_hs_stream_batch<true, true><<<B, HS_THREADS, smem, p->stream>>>(p->P, F);
    else k_hs_stream_batch<false, true><<<B, HS_THREADS, smem, p->stream>>>(p->P, F);
  } else {
    if (p->P.exact) k_hs_stream_batch<true, false><<<B, HS_THREADS, smem, p->stream>>>(p->P, F);
    else k_hs_stream_batch<false, false><<<B, HS_THREADS, smem, p->stream>>>(p->P, F);
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  std::vector<float> host(16 * T);
  B2S_CUDA_CHECK(cudaMemcpyAsync(host.data(), d_out, sizeof(float) * 16 * T, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  for (size_t i = 0; i < T; i++) {
    std::memcpy(out_poses + 3 * i, host.data() + 16 * i, 3 * sizeof(float));
    if (out_map_updated) out_map_updated[i] = host[16 * i + 12] != 0.0f ? 1 : 0;
    if (out_n_points) std::memcpy(out_n_points + i, host.data() + 16 * i + 15, sizeof(int32_t));  // (ingest) kept beams
  }
  if (out_last_covs && !map_without_matching)
    for (int b = 0; b < B; b++)
      if (n_scans[b] > 0) std::memcpy(out_last_covs + 9 * (size_t)b, host.data() + 16 * (size_t)(first[2 * (size_t)b + 1] - 1) + 3, 9 * sizeof(float));
  return B2S_OK;
}

// One batched step on the processor's stream: k_hs_match of scan b = the d_n_points[b] points at d_points + 2 b cap,
// then the grid-wide map update passes (k_hs_mark, k_hs_apply); max_n is the step's largest point count
static b2s_status hs_launch_step(b2s_hector_slam *p, const float *d_points, const int32_t *d_n_points, int max_n,
                                 const float origo[2], const float *d_pose_hints, int map_without_matching) {
  const int B = p->batch;
  HsCall C;
  std::memset(&C, 0, sizeof(C));
  C.pts0 = d_points; C.n0 = d_n_points; C.pts_stride = p->cap;
  C.hints = d_pose_hints;
  C.origo_x = origo[0]; C.origo_y = origo[1];
  C.map_without_matching = map_without_matching;
  C.out = p->d_out;
  if (p->P.exact) k_hs_match<true><<<B, HS_THREADS, hs_smem_bytes(p->cap), p->stream>>>(p->P, C);
  else k_hs_match<false><<<B, HS_THREADS, hs_smem_bytes(p->cap), p->stream>>>(p->P, C);
  // data containers of the coarse levels may hold more points than this step's scans (map_without_matching): size the
  // update grid by the capacity bound
  const dim3 grid(std::max(1, std::min(ceil_div(std::max(max_n, 1) * p->levels, 8), sm_count(p->device) * 8 / std::max(1, std::min(B, 8)))), grid_rows(B));
  k_hs_mark<<<grid, 256, 0, p->stream>>>(p->P);
  k_hs_apply<<<grid, 256, 0, p->stream>>>(p->P);
  B2S_CUDA_CHECK(cudaGetLastError());
  return B2S_OK;
}

// k_hs_stream_batch<_, true>'s input in device memory, freed in stream order with the caller: the ranges, the unit
// vectors, and one block holding the HsIngest (`ingest`), then the B lasers, then the B level-0 origos
struct HsIngestUpload {
  AsyncBuf<float> ranges;
  AsyncBuf<double> units;
  AsyncBuf<unsigned char> block;
  const HsIngest *ingest = nullptr;
  explicit HsIngestUpload(cudaStream_t s) : ranges(s), units(s), block(s) {}
};

// Uploads the call's n_floats ranges, n_units unit vectors ([n_units][2]) and processor b's laser lasers[b], and
// writes each processor's level-0 origo: dataContainer.setOrigo (hector_slam.cc:329) of its mount, the same on every
// scan, which the ingest kernel's match reads there (hs_match_cta<_, _, true>) instead of a per-CTA value held through
// the scan loop.  The origo of a processor without scans in the call is not read before it is written again: every
// other match writes origo[0] before reading it, and every ingest launch follows this call's write.
// The descriptor, the lasers and the origos travel in ONE copy from pageable memory (each such copy is staged by the
// host before it returns, several microseconds that a call per scan pays every scan); the origos then reach the
// processors' states by a copy on the device.
static b2s_status hs_ingest_upload(b2s_hector_slam *p, HsIngestUpload &d, size_t n_floats, const float *ranges,
                                   size_t n_units, const double *units, const HsLaser *lasers) {
  static_assert(sizeof(HsIngest) % alignof(HsLaser) == 0 && sizeof(HsLaser) % alignof(float2) == 0,
                "the block's parts stay aligned");
  const int B = p->batch;
  const size_t at_lasers = sizeof(HsIngest), at_origo = at_lasers + sizeof(HsLaser) * (size_t)B;
  const size_t bytes = at_origo + sizeof(float2) * (size_t)B;
  B2S_CUDA_CHECK(d.ranges.alloc(std::max<size_t>(n_floats, 1)));
  B2S_CUDA_CHECK(d.units.alloc(2 * std::max<size_t>(n_units, 1)));
  B2S_CUDA_CHECK(d.block.alloc(bytes));
  std::vector<unsigned char> h(bytes);
  HsIngest I;
  std::memset(&I, 0, sizeof(I));
  I.ranges = d.ranges;
  I.units = reinterpret_cast<const double2 *>(static_cast<double *>(d.units));
  I.lasers = reinterpret_cast<const HsLaser *>(d.block.p + at_lasers);
  std::memcpy(h.data(), &I, sizeof(I));
  std::memcpy(h.data() + at_lasers, lasers, sizeof(HsLaser) * (size_t)B);
  for (int b = 0; b < B; b++) {
    const HectorBeamFilter &f = lasers[b].filter;
    const float2 o = make_float2((float)f.mount.o[0] * f.scale_to_map, (float)f.mount.o[1] * f.scale_to_map);
    std::memcpy(h.data() + at_origo + sizeof(float2) * (size_t)b, &o, sizeof(o));
  }
  // (pageable sources: staged before the calls return)
  if (n_floats > 0) B2S_CUDA_CHECK(cudaMemcpyAsync(d.ranges, ranges, sizeof(float) * n_floats, cudaMemcpyHostToDevice, p->stream));
  if (n_units > 0) B2S_CUDA_CHECK(cudaMemcpyAsync(d.units, units, sizeof(double) * 2 * n_units, cudaMemcpyHostToDevice, p->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d.block, h.data(), bytes, cudaMemcpyHostToDevice, p->stream));
  B2S_CUDA_CHECK(cudaMemcpy2DAsync(&p->d_state.p[0].origo[0][0], sizeof(HsState), d.block.p + at_origo, sizeof(float2),
                                   sizeof(float2), (size_t)B, cudaMemcpyDeviceToDevice, p->stream));
  d.ingest = reinterpret_cast<const HsIngest *>(d.block.p);
  return B2S_OK;
}

namespace b2s {

// HectorMappingRos::setMapInfo (hector_slam.cc:165-180) of processor b's level 0: getWorldCoords(0, 0) - cell length * 0.5f
void hs_node_map_info(const b2s_hector_slam *p, int b, float &origin_x, float &origin_y, float &cell_length, int &w, int &h) {
  const HsLevel &m = p->procs[(size_t)b].l[0];
  float wx, wy;
  get_world_coords(m.tf, 0.0f, 0.0f, wx, wy);
  cell_length = p->specs[(size_t)b].map_resolution;
  origin_x = wx - cell_length * 0.5f;
  origin_y = wy - cell_length * 0.5f;
  w = m.sx;
  h = m.sy;
}

// GridMapBase::getScaleToMap of processor b's level 0
float hs_scale_to_map(const b2s_hector_slam *p, int b) { return p->procs[(size_t)b].l[0].tf.tw_lin; }

// ---- lesson4's HectorMappingRos (hector_node.cu): one node per processor, over one call ----
struct HsRosJob {  // one node's level-0 plane -> its ROS payload at `out` in a slot
  const float *lo;
  long long out;
  int cells;
};
// the publishes before one part: job blockIdx.y converts its node's cells (nodes of any map size, back to back)
static __global__ void k_hector_ros_nodes(const HsRosJob *__restrict__ jobs, int8_t *__restrict__ out) {
  const HsRosJob J = jobs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= J.cells) return;
  out[J.out + i] = hector_ros_cell(J.lo[i]);
}

// The call runs as the plan's parts (hector_node_plan.cuh), one k_hs_stream_batch<true, true> launch of B CTAs per
// part that has scans, CTA b on node b's scans of the part.  Before part k >= 1, one k_hector_ros_nodes launch on the
// processor's stream converts level 0 of every node publishing there into one slot of payloads, back to back; a second
// stream copies the slot, with those nodes' record rows of part k - 1, into page-locked memory while part k's launch
// runs.  Two slots, each as large as the most cells published before one part: a slot is handed to on_map (part by
// part, nodes ascending inside a part) before it is converted into again.  on_map(b, k, payload, rows, n) also gets
// node b's n record rows since its previous publish.  Node b's scans are n_scans[b] rows of lasers[b].n_ranges floats
// (lasers[b].base is set here), node-major; units holds every laser's unit vectors.  Rows are node-major throughout.
b2s_status hs_node_run(b2s_hector_slam *p, HsNodeIo &io, const HsLaser *lasers, const double *units, size_t n_units,
                       const HectorNodePlan &plan, const int32_t *n_scans, const float *ranges, float *out_rows,
                       const std::function<b2s_status(int, int, const int8_t *, const float *, long long)> &on_map) {
  const int B = plan.batch, K = plan.n_parts;
  // parts [K][B] = node b's scans [first, end) of part k, node-major over the call
  std::vector<long long> parts(2 * (size_t)K * B);
  std::vector<HsLaser> las(lasers, lasers + B);
  long long first = 0, floats = 0;
  int longest = 0;
  for (int b = 0; b < B; b++) {
    for (int k = 0; k < K; k++) {
      const size_t e = (size_t)k * B + b;
      parts[2 * e] = first + plan.begin[e];
      parts[2 * e + 1] = first + plan.end[e];
    }
    las[(size_t)b].base = floats - first * las[(size_t)b].n_ranges;
    first += n_scans[b];
    floats += (long long)n_scans[b] * las[(size_t)b].n_ranges;
    longest = std::max(longest, (int)n_scans[b]);
  }
  const size_t T = (size_t)first;
  // the nodes publishing before part k: jobs[pub0[k] .. pub0[k + 1]) (nodes pub[...]), those with k publishes or more,
  // ascending, each at its offset in the part's slot
  std::vector<int> pub;
  std::vector<HsRosJob> jobs;
  std::vector<size_t> pub0((size_t)K + 1, 0);
  std::vector<int> widest((size_t)K, 0);  // the most cells of one node publishing before part k
  long long most = 0;
  for (int k = 0; k < K; k++) {
    long long at = 0;
    for (int b = 0; k > 0 && b < B; b++)
      if ((int)plan.cuts[(size_t)b].size() >= k) {
        const HsLevel &m = p->procs[(size_t)b].l[0];
        const int cells = m.sx * m.sy;
        pub.push_back(b);
        jobs.push_back(HsRosJob{m.lo, at, cells});
        at += cells;
        widest[(size_t)k] = std::max(widest[(size_t)k], cells);
      }
    pub0[(size_t)k + 1] = pub.size();
    most = std::max(most, at);
  }
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  if ((st = hs_reserve_epochs(p, (unsigned long long)longest))) return st;  // per processor: its own scans
  B2S_CUDA_CHECK(io.h_rows.reserve(16 * T));
  if (most > 0)  // the first call that publishes allocates the slots; later calls reuse them (or grow them)
    for (int s = 0; s < 2; s++) {
      B2S_CUDA_CHECK(io.d_map[s].reserve((size_t)most));
      B2S_CUDA_CHECK(io.h_map[s].reserve((size_t)most));
    }
  HsIngestUpload d_in(p->stream);
  AsyncBuf<float> d_out(p->stream);
  AsyncBuf<long long> d_parts(p->stream);
  AsyncBuf<HsRosJob> d_jobs(p->stream);
  B2S_CUDA_CHECK(d_parts.alloc(parts.size()));
  B2S_CUDA_CHECK(d_jobs.alloc(std::max<size_t>(jobs.size(), 1)));
  B2S_CUDA_CHECK(d_out.alloc(16 * std::max<size_t>(T, 1)));
  if ((st = hs_ingest_upload(p, d_in, (size_t)floats, ranges, n_units, units, las.data()))) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_parts, parts.data(), sizeof(long long) * parts.size(), cudaMemcpyHostToDevice, p->stream));
  if (!jobs.empty()) B2S_CUDA_CHECK(cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(HsRosJob) * jobs.size(), cudaMemcpyHostToDevice, p->stream));
  // the copy stream reads d_out: on every way out it is drained before the stream-ordered frees above
  struct DrainCopies {
    cudaStream_t s;
    ~DrainCopies() { cudaStreamSynchronize(s); }
  } drain_copies{io.copy};
  HsFleet F;
  std::memset(&F, 0, sizeof(F));
  F.ingest = d_in.ingest;
  F.out = d_out;
  const size_t smem = hs_smem_bytes(p->cap);
  struct Pending { int k, slot; };
  std::vector<Pending> pending;
  int slot = 0;
  auto drain_one = [&]() -> b2s_status {
    const Pending q = pending.front();
    pending.erase(pending.begin());
    B2S_CUDA_CHECK(cudaEventSynchronize(io.copied[q.slot]));
    for (size_t j = pub0[(size_t)q.k]; j < pub0[(size_t)q.k + 1]; j++) {
      const long long *prev = parts.data() + 2 * ((size_t)(q.k - 1) * B + pub[j]);  // the rows before this publish
      if (b2s_status s = on_map(pub[j], q.k, io.h_map[q.slot] + jobs[j].out, io.h_rows + 16 * prev[0], prev[1] - prev[0]))
        return s;
    }
    return B2S_OK;
  };
  for (int k = 0; k < K; k++) {
    const size_t np = pub0[(size_t)k + 1] - pub0[(size_t)k];
    if (np > 0) {  // the publishes before part k (k >= 1)
      if (pending.size() == 2) {
        if ((st = drain_one())) return st;
      }
      const HsRosJob &last = jobs[pub0[(size_t)k + 1] - 1];
      k_hector_ros_nodes<<<dim3((unsigned)ceil_div((long long)widest[(size_t)k], 256), (unsigned)np), 256, 0, p->stream>>>(
          d_jobs + pub0[(size_t)k], io.d_map[slot]);
      B2S_CUDA_CHECK(cudaGetLastError());
      B2S_CUDA_CHECK(cudaEventRecord(io.converted[slot], p->stream));
      B2S_CUDA_CHECK(cudaStreamWaitEvent(io.copy, io.converted[slot], 0));
      B2S_CUDA_CHECK(cudaMemcpyAsync(io.h_map[slot], io.d_map[slot], (size_t)(last.out + last.cells), cudaMemcpyDeviceToHost,
                                     io.copy));
      for (size_t j = pub0[(size_t)k]; j < pub0[(size_t)k + 1]; j++) {
        const long long *prev = parts.data() + 2 * ((size_t)(k - 1) * B + pub[j]);
        if (prev[1] > prev[0])
          B2S_CUDA_CHECK(cudaMemcpyAsync(io.h_rows + 16 * prev[0], d_out + 16 * prev[0],
                                         sizeof(float) * 16 * (size_t)(prev[1] - prev[0]), cudaMemcpyDeviceToHost, io.copy));
      }
      B2S_CUDA_CHECK(cudaEventRecord(io.copied[slot], io.copy));
      pending.push_back(Pending{k, slot});
      slot ^= 1;
    }
    long long scans = 0;
    for (int b = 0; b < B; b++) scans += parts[2 * ((size_t)k * B + b) + 1] - parts[2 * ((size_t)k * B + b)];
    if (scans > 0) {
      F.first = d_parts + 2 * (size_t)k * B;
      k_hs_stream_batch<true, true><<<B, HS_THREADS, smem, p->stream>>>(p->P, F);
      B2S_CUDA_CHECK(cudaGetLastError());
    }
  }
  while (!pending.empty())
    if ((st = drain_one())) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(out_rows, d_out, sizeof(float) * 16 * T, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(io.copy));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  return B2S_OK;
}

}  // namespace b2s

extern "C" {

b2s_status b2s_hector_slam_create(float map_resolution, int map_size_x, int map_size_y, float start_x, float start_y,
                                  int levels, int device, void *cuda_stream, b2s_hector_slam **out) {
  const b2s_hector_map_spec s = hs_default_spec(map_resolution, map_size_x, map_size_y, start_x, start_y, levels);
  return hs_create(1, 2048, &s, device, cuda_stream, out, "b2s_hector_slam_create");
}

b2s_status b2s_hector_slam_create_batch(int batch, int max_points, float map_resolution, int map_size_x, int map_size_y,
                                        float start_x, float start_y, int levels, int device, void *cuda_stream,
                                        b2s_hector_slam **out) {
  if (batch < 1) return hs_create(batch, max_points, nullptr, device, cuda_stream, out, "b2s_hector_slam_create_batch");
  const std::vector<b2s_hector_map_spec> specs(
      (size_t)batch, hs_default_spec(map_resolution, map_size_x, map_size_y, start_x, start_y, levels));
  return hs_create(batch, max_points, specs.data(), device, cuda_stream, out, "b2s_hector_slam_create_batch");
}

b2s_status b2s_hector_slam_create_fleet(int batch, int max_points, const b2s_hector_map_spec *maps, int device,
                                        void *cuda_stream, b2s_hector_slam **out) {
  return hs_create(batch, max_points, maps, device, cuda_stream, out, "b2s_hector_slam_create_fleet");
}

void b2s_hector_slam_destroy(b2s_hector_slam *p) {
  if (!p) return;
  cudaSetDevice(p->device);
  cudaStreamSynchronize(p->stream);
  delete p;
}

b2s_status b2s_hector_slam_set_update_factors(b2s_hector_slam *p, float update_free, float update_occupied) {
  if (!p) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  for (HsProc &q : p->procs) {
    q.lo_free = prob_to_log_odds(update_free);
    q.lo_occ = prob_to_log_odds(update_occupied);
  }
  return hs_upload_procs(p);
}

b2s_status b2s_hector_slam_set_map_update_min_diff(b2s_hector_slam *p, float min_dist, float min_angle) {
  if (!p) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  for (HsProc &q : p->procs) {
    q.min_dist = min_dist;
    q.min_angle = min_angle;
  }
  return hs_upload_procs(p);
}

b2s_status b2s_hector_slam_set_exact(b2s_hector_slam *p, int exact) {
  if (!p) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  p->P.exact = exact ? 1 : 0;
  return B2S_OK;
}

int32_t b2s_hector_slam_match_cluster_size(const b2s_hector_slam *p) { return p ? (int32_t)p->cluster : 0; }

b2s_status b2s_hector_slam_reset(b2s_hector_slam *p) {
  if (!p) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  k_hs_state_init<<<ceil_div(p->batch, 128), 128, 0, p->stream>>>(p->d_state, p->batch, 1);
  return hs_clear_maps(p);
}

b2s_status b2s_hector_slam_update(b2s_hector_slam *p, const float *points, int n_points, const float origo[2],
                                  const float pose_hint_world[3], int map_without_matching, float out_pose[3],
                                  float out_cov[9], int *out_map_updated) {
  B2S_NVTX("Hector update (match + gate + map update)");
  if (!p || !origo || !pose_hint_world || !out_pose || n_points < 0 || (n_points > 0 && !points))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (p->batch != 1) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_slam_update serves single-processor handles; use b2s_hector_slam_update_batch");
  if (n_points > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "more points than the handle's capacity (2048 for b2s_hector_slam_create)");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);  // the previous call's update passes still read nothing of ours, but its kernel reads h_hint / h_pts
  if (st) return st;
  if ((st = hs_reserve_epochs(p, 1))) return st;
  if (n_points > 0) std::memcpy(p->h_pts, points, sizeof(float) * 2 * (size_t)n_points);
  p->h_hint[0] = pose_hint_world[0]; p->h_hint[1] = pose_hint_world[1]; p->h_hint[2] = pose_hint_world[2];
  p->seq += 1;
  if (p->seq == 0) p->seq = 1;
  HsStream S;
  std::memset(&S, 0, sizeof(S));
  S.pts = p->h_pts.dev;        // read over the host link by the matching CTA (8.6 KB for 1081 beams)
  S.count0 = n_points;
  S.n_scans = 1;
  S.first_hint = p->h_hint.dev;
  S.origo_x = origo[0]; S.origo_y = origo[1];
  S.map_without_matching = map_without_matching;
  S.out = p->d_out;
  S.mailbox = p->h_mail.dev;
  S.seq = p->seq;
  if ((st = hs_launch_stream(p, S))) return st;
  B2S_CUDA_CHECK(cudaEventRecord(p->ev_done, p->stream));
  p->launch_pending = true;
  // the pose arrives through the mailbox as soon as the match is done; the update passes keep running
  const volatile unsigned int *flag = reinterpret_cast<const volatile unsigned int *>(p->h_mail.p) + 15;
  for (unsigned long long spin = 0;; spin++) {
    if (*flag == p->seq) break;
    if ((spin & 0x3fff) == 0x3fff) {
      const cudaError_t q = cudaEventQuery(p->ev_done);
      if (q == cudaSuccess) {
        if (*flag == p->seq) break;
        B2S_FAIL(B2S_ERR_CUDA, "b2s_hector_slam_update: the kernel finished without posting its result");
      }
      if (q != cudaErrorNotReady) B2S_CUDA_CHECK(q);
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  float r[15];
  for (int q = 0; q < 15; q++) r[q] = p->h_mail[q];
  if (r[14] != 0.0f) B2S_FAIL(B2S_ERR_CUDA, "b2s_hector_slam_update: a cluster exchange of the match timed out");
  out_pose[0] = r[0]; out_pose[1] = r[1]; out_pose[2] = r[2];
  if (out_cov && !map_without_matching) std::memcpy(out_cov, r + 3, 9 * sizeof(float));
  if (out_map_updated) *out_map_updated = r[12] != 0.0f ? 1 : 0;
  return B2S_OK;
}

b2s_status b2s_hector_slam_process_stream(b2s_hector_slam *p, int n_scans, const float *points, const int32_t *n_points,
                                          const float origo[2], const float *first_pose_hint, const float *pose_hints,
                                          int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                          float *out_last_cov) {
  B2S_NVTX("Hector stream");
  if (!p || n_scans < 0 || !origo || !out_poses || (n_scans > 0 && (!points || !n_points)))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (map_without_matching && !pose_hints) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map_without_matching needs a pose per scan (pose_hints)");
  if (p->batch != 1) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_hector_slam_process_stream serves single-processor handles");
  if (n_scans == 0) return B2S_OK;
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  std::vector<int> offs((size_t)n_scans);
  long long total = 0;
  for (int i = 0; i < n_scans; i++) {
    if (n_points[i] < 0 || n_points[i] > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "a scan has more points than the handle's capacity");
    offs[i] = (int)total;
    total += n_points[i];
    if (total > 0x7fffffffLL / 2) B2S_FAIL(B2S_ERR_TOO_LARGE, "stream too long for one call");
  }
  if ((st = hs_reserve_epochs(p, (unsigned long long)n_scans))) return st;
  AsyncBuf<float> d_pts(p->stream), d_hints(p->stream), d_first(p->stream), d_out(p->stream);
  AsyncBuf<int> d_offs(p->stream), d_cnt(p->stream);
  B2S_CUDA_CHECK(d_pts.alloc(2 * (size_t)std::max<long long>(total, 1)));
  B2S_CUDA_CHECK(d_out.alloc(16 * (size_t)n_scans));
  B2S_CUDA_CHECK(cudaMemsetAsync(d_out, 0, sizeof(float) * 16 * (size_t)n_scans, p->stream));  // no stale verdict tags
  B2S_CUDA_CHECK(d_offs.alloc(n_scans));
  B2S_CUDA_CHECK(d_cnt.alloc(n_scans));
  if (total > 0) B2S_CUDA_CHECK(cudaMemcpyAsync(d_pts, points, sizeof(float) * 2 * (size_t)total, cudaMemcpyHostToDevice, p->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_offs, offs.data(), sizeof(int) * (size_t)n_scans, cudaMemcpyHostToDevice, p->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_cnt, n_points, sizeof(int) * (size_t)n_scans, cudaMemcpyHostToDevice, p->stream));
  if (pose_hints) {
    B2S_CUDA_CHECK(d_hints.alloc(3 * (size_t)n_scans));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_hints, pose_hints, sizeof(float) * 3 * (size_t)n_scans, cudaMemcpyHostToDevice, p->stream));
  } else if (first_pose_hint) {
    B2S_CUDA_CHECK(d_first.alloc(3));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_first, first_pose_hint, sizeof(float) * 3, cudaMemcpyHostToDevice, p->stream));
  }
  HsStream S;
  std::memset(&S, 0, sizeof(S));
  S.pts = d_pts; S.offsets = d_offs; S.counts = d_cnt; S.n_scans = n_scans;
  S.hints = d_hints; S.first_hint = d_first;
  S.origo_x = origo[0]; S.origo_y = origo[1];
  S.map_without_matching = map_without_matching;
  S.out = d_out;
  if ((st = hs_launch_stream(p, S))) return st;
  std::vector<float> host((size_t)n_scans * 16);
  B2S_CUDA_CHECK(cudaMemcpyAsync(host.data(), d_out, sizeof(float) * 16 * (size_t)n_scans, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  for (int i = 0; i < n_scans; i++) {
    if (host[16 * (size_t)i + 14] != 0.0f) B2S_FAIL(B2S_ERR_CUDA, "b2s_hector_slam_process_stream: a cluster exchange of the match timed out");
    std::memcpy(out_poses + 3 * (size_t)i, host.data() + 16 * (size_t)i, 3 * sizeof(float));
    if (out_map_updated) out_map_updated[i] = host[16 * (size_t)i + 12] != 0.0f ? 1 : 0;
  }
  if (out_last_cov && !map_without_matching) std::memcpy(out_last_cov, host.data() + 16 * (size_t)(n_scans - 1) + 3, 9 * sizeof(float));
  return B2S_OK;
}

b2s_status b2s_hector_slam_process_stream_batch(b2s_hector_slam *p, const int32_t *n_scans, const float *points,
                                                const int32_t *n_points, const float origo[2],
                                                const float *first_pose_hints, const float *pose_hints,
                                                int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                                float *out_last_covs) {
  B2S_NVTX("Hector batched streams");
  if (!p || !n_scans || !origo || !out_poses) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (map_without_matching && !pose_hints) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map_without_matching needs a pose per scan (pose_hints)");
  // every count is checked before anything is enqueued: a refused call changes nothing
  std::vector<long long> first;
  int longest = 0;
  b2s_status st = hs_fleet_counts(p, n_scans, first, longest);
  if (st) return st;
  const long long total = first.back();
  if (total > 0 && (!points || !n_points)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if ((unsigned)longest >= HS_EPOCH_MAX) B2S_FAIL(B2S_ERR_TOO_LARGE, "too many scans of one processor in one call (stamp epochs are 20 bits)");
  std::vector<long long> offs((size_t)total);
  long long n_pts = 0;
  for (long long i = 0; i < total; i++) {
    if (n_points[i] < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "negative point count");
    if (n_points[i] > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "a scan has more points than the handle's capacity");
    offs[(size_t)i] = n_pts;
    n_pts += n_points[i];
  }
  AsyncBuf<float> d_pts(p->stream);
  AsyncBuf<long long> d_offs(p->stream);
  AsyncBuf<int> d_cnt(p->stream);
  auto upload = [&](HsFleet &F) -> b2s_status {
    const size_t T = (size_t)total;
    B2S_CUDA_CHECK(d_pts.alloc(2 * (size_t)std::max<long long>(n_pts, 1)));
    B2S_CUDA_CHECK(d_offs.alloc(T));
    B2S_CUDA_CHECK(d_cnt.alloc(T));
    if (n_pts > 0) B2S_CUDA_CHECK(cudaMemcpyAsync(d_pts, points, sizeof(float) * 2 * (size_t)n_pts, cudaMemcpyHostToDevice, p->stream));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_offs, offs.data(), sizeof(long long) * T, cudaMemcpyHostToDevice, p->stream));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_cnt, n_points, sizeof(int) * T, cudaMemcpyHostToDevice, p->stream));
    F.pts = d_pts; F.offsets = d_offs; F.counts = d_cnt;
    F.origo_x = origo[0]; F.origo_y = origo[1];
    return B2S_OK;
  };
  return hs_fleet_run(p, n_scans, first, longest, false, first_pose_hints, pose_hints, map_without_matching, out_poses,
                      out_map_updated, out_last_covs, nullptr, upload);
}

b2s_status b2s_hector_slam_process_scans_batch(b2s_hector_slam *p, const b2s_laser_scan_msg *geometry,
                                               const b2s_hector_scan_filter *filter, const int32_t *n_scans,
                                               const float *ranges, const float *first_pose_hints, const float *pose_hints,
                                               int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                               float *out_last_covs, int32_t *out_n_points) {
  B2S_NVTX("Hector batched LaserScan streams");
  if (!p || !geometry || !filter || !n_scans || !out_poses || geometry->n_ranges < 0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument or negative count");
  if (map_without_matching && !pose_hints) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map_without_matching needs a pose per scan (pose_hints)");
  const int n = geometry->n_ranges;
  if (n > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "more ranges per scan than the handle's capacity");
  const int B = p->batch;
  std::vector<long long> first;
  int longest = 0;
  b2s_status st = hs_fleet_counts(p, n_scans, first, longest);
  if (st) return st;
  const long long total = first.back();
  if (total > 0 && n > 0 && !ranges) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if ((unsigned)longest >= HS_EPOCH_MAX) B2S_FAIL(B2S_ERR_TOO_LARGE, "too many scans of one processor in one call (stamp epochs are 20 bits)");
  // one laser for every processor (base 0: scan i's ranges are row i), each scaled to its own level 0
  const b2s_hector_scan_filter &q = *filter;
  std::vector<HsLaser> lasers((size_t)B);
  for (int b = 0; b < B; b++) {
    HsLaser &l = lasers[(size_t)b];
    l.filter = hector_scan_filter(q.laser_in_base, hs_scale_to_map(p, b), q.min_dist, q.max_dist, q.use_max_scan_range,
                                  q.z_min, q.z_max);
    l.base = 0;
    l.unit0 = 0;
    l.n_ranges = n;
    l.range_min = geometry->range_min;
    l.range_cutoff = hector_range_cutoff(q.range_cutoff, geometry->range_max);
  }
  std::vector<double> unit(2 * (size_t)n);
  hector_unit_vectors(geometry->angle_min, geometry->angle_increment, n, unit.data());
  HsIngestUpload d_in(p->stream);
  auto upload = [&](HsFleet &F) -> b2s_status {
    if (b2s_status s = hs_ingest_upload(p, d_in, (size_t)total * (size_t)n, ranges, (size_t)n, unit.data(), lasers.data()))
      return s;
    F.ingest = d_in.ingest;
    return B2S_OK;
  };
  return hs_fleet_run(p, n_scans, first, longest, true, first_pose_hints, pose_hints, map_without_matching, out_poses,
                      out_map_updated, out_last_covs, out_n_points, upload);
}

b2s_status b2s_hector_slam_update_batch(b2s_hector_slam *p, const float *points, const int32_t *n_points, const float origo[2],
                                        const float *pose_hints, int map_without_matching, float *out_poses, float *out_covs,
                                        int32_t *out_map_updated) {
  if (!p || !points || !n_points || !origo || !out_poses) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (map_without_matching && !pose_hints) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map_without_matching needs the poses (pose_hints)");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  const int B = p->batch;
  for (int b = 0; b < B; b++)
    if (n_points[b] < 0 || n_points[b] > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "a scan has more points than the handle's capacity");
  if ((st = hs_reserve_epochs(p, 1))) return st;
  AsyncBuf<float> d_pts(p->stream), d_hints(p->stream);
  AsyncBuf<int> d_cnt(p->stream);
  B2S_CUDA_CHECK(d_pts.alloc(2 * (size_t)p->cap * B));
  B2S_CUDA_CHECK(d_cnt.alloc(B));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_pts, points, sizeof(float) * 2 * (size_t)p->cap * B, cudaMemcpyHostToDevice, p->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(d_cnt, n_points, sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, p->stream));
  if (pose_hints) {
    B2S_CUDA_CHECK(d_hints.alloc(3 * (size_t)B));
    B2S_CUDA_CHECK(cudaMemcpyAsync(d_hints, pose_hints, sizeof(float) * 3 * (size_t)B, cudaMemcpyHostToDevice, p->stream));
  }
  int max_n = 0;
  for (int b = 0; b < B; b++) max_n = std::max(max_n, n_points[b]);
  if ((st = hs_launch_step(p, d_pts, d_cnt, max_n, origo, d_hints, map_without_matching))) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(p->h_out, p->d_out, sizeof(float) * 16 * (size_t)B, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  for (int b = 0; b < B; b++) {
    std::memcpy(out_poses + 3 * (size_t)b, p->h_out + 16 * (size_t)b, 3 * sizeof(float));
    if (out_covs && !map_without_matching) std::memcpy(out_covs + 9 * (size_t)b, p->h_out + 16 * (size_t)b + 3, 9 * sizeof(float));
    if (out_map_updated) out_map_updated[b] = p->h_out[16 * (size_t)b + 12] != 0.0f ? 1 : 0;
  }
  return B2S_OK;
}

/* the same step with the scans ALREADY on the device (device pointers; nothing is copied, nothing is returned to the
 * host): the resident-in-HBM form the throughput of the batched update is measured on */
b2s_status b2s_hector_slam_update_batch_device(b2s_hector_slam *p, const float *d_points, const int32_t *d_n_points, int max_n,
                                               const float origo[2], const float *d_pose_hints, int map_without_matching) {
  B2S_NVTX("Hector batch step");
  if (!p || !d_points || !d_n_points || !origo) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (map_without_matching && !d_pose_hints) B2S_FAIL(B2S_ERR_BAD_PARAMS, "map_without_matching needs the poses");
  if (max_n < 0 || max_n > p->cap) B2S_FAIL(B2S_ERR_TOO_LARGE, "more points than the handle's capacity");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  b2s_status st = hs_wait_launch(p);
  if (st) return st;
  if ((st = hs_reserve_epochs(p, 1))) return st;
  return hs_launch_step(p, d_points, d_n_points, max_n, origo, d_pose_hints, map_without_matching);
}

b2s_status b2s_hector_slam_sync(b2s_hector_slam *p) {
  if (!p) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  p->launch_pending = false;
  return B2S_OK;
}

b2s_status b2s_hector_slam_level_dims_of(b2s_hector_slam *p, int b, int level, int dims[2], float *cell_length) {
  if (!p || !dims || b < 0 || b >= p->batch || level < 0 || level >= p->procs[(size_t)b].levels)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad level / processor");
  dims[0] = p->procs[(size_t)b].l[level].sx;
  dims[1] = p->procs[(size_t)b].l[level].sy;
  if (cell_length) *cell_length = hs_cell_length(p->specs[(size_t)b], level);
  return B2S_OK;
}

b2s_status b2s_hector_slam_level_dims(b2s_hector_slam *p, int level, int dims[2], float *cell_length) {
  return b2s_hector_slam_level_dims_of(p, 0, level, dims, cell_length);
}

b2s_status b2s_hector_slam_copy_level_of(b2s_hector_slam *p, int b, int level, float *log_odds, int32_t *update_index) {
  if (!p || b < 0 || b >= p->batch || level < 0 || level >= p->procs[(size_t)b].levels)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad level / processor");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  const HsLevel &m = p->procs[(size_t)b].l[level];
  const size_t cells = (size_t)m.sx * m.sy;
  if (log_odds) B2S_CUDA_CHECK(cudaMemcpyAsync(log_odds, m.lo, cells * 4, cudaMemcpyDeviceToHost, p->stream));
  if (update_index) B2S_CUDA_CHECK(cudaMemcpyAsync(update_index, m.ui, cells * 4, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  p->launch_pending = false;
  return B2S_OK;
}

b2s_status b2s_hector_slam_copy_level(b2s_hector_slam *p, int level, float *log_odds, int32_t *update_index) {
  return b2s_hector_slam_copy_level_of(p, 0, level, log_odds, update_index);
}

b2s_status b2s_hector_slam_copy_level_ros_of(b2s_hector_slam *p, int b, int level, int8_t *out) {
  if (!p || !out || b < 0 || b >= p->batch || level < 0 || level >= p->procs[(size_t)b].levels)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad level / processor");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  const HsLevel &m = p->procs[(size_t)b].l[level];
  const int n = m.sx * m.sy;
  AsyncBuf<int8_t> d(p->stream);
  B2S_CUDA_CHECK(d.alloc((size_t)n));
  k_hector_ros<<<ceil_div(n, 256), 256, 0, p->stream>>>(m.lo, n, d);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, d, (size_t)n, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  p->launch_pending = false;
  return B2S_OK;
}

b2s_status b2s_hector_slam_copy_level_ros(b2s_hector_slam *p, int level, int8_t *out) {
  return b2s_hector_slam_copy_level_ros_of(p, 0, level, out);
}

b2s_status b2s_hector_slam_stats(b2s_hector_slam *p, double out[5]) {
  if (!p || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  std::vector<HsState> s((size_t)p->batch);
  B2S_CUDA_CHECK(cudaMemcpyAsync(s.data(), p->d_state, sizeof(HsState) * (size_t)p->batch, cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  p->launch_pending = false;
  out[0] = out[1] = out[2] = 0.0;
  for (const HsState &x : s) { out[0] += (double)x.n_matched; out[1] += (double)x.n_updated; out[2] += (double)x.visits; }
  out[3] = (double)s[0].t_match_ns * 1e-6;   // ms of processor 0's last match / update (device %globaltimer)
  out[4] = (double)s[0].t_update_ns * 1e-6;
  return B2S_OK;
}

/* the processor's own last poses (getLastScanMatchPose / getLastMapUpdatePose, HectorSlamProcessor.h:118-119) */
b2s_status b2s_hector_slam_last_poses(b2s_hector_slam *p, int b, float last_scan_match_pose[3], float last_map_update_pose[3]) {
  if (!p || b < 0 || b >= p->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad processor");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  HsState s;
  B2S_CUDA_CHECK(cudaMemcpyAsync(&s, p->d_state + b, sizeof(HsState), cudaMemcpyDeviceToHost, p->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  p->launch_pending = false;
  if (last_scan_match_pose) std::memcpy(last_scan_match_pose, s.last_match_pose, 3 * sizeof(float));
  if (last_map_update_pose) std::memcpy(last_map_update_pose, s.last_update_pose, 3 * sizeof(float));
  return B2S_OK;
}

/* test hook: pretend `updates` map updates have already consumed stamp epochs (exercises the 20-bit epoch wrap) */
b2s_status b2s_hector_slam_debug_set_epoch(b2s_hector_slam *p, unsigned int updates) {
  if (!p || updates >= HS_EPOCH_MAX) B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad epoch");
  B2S_CUDA_CHECK(cudaSetDevice(p->device));
  B2S_CUDA_CHECK(cudaStreamSynchronize(p->stream));
  std::vector<HsState> s((size_t)p->batch);
  B2S_CUDA_CHECK(cudaMemcpy(s.data(), p->d_state, sizeof(HsState) * (size_t)p->batch, cudaMemcpyDeviceToHost));
  unsigned int have = 0;
  for (const HsState &x : s)
    for (int l = 0; l < p->levels; l++) have = std::max(have, x.epoch[l]);
  if (updates < have) B2S_FAIL(B2S_ERR_BAD_PARAMS, "epochs only move forward");
  for (HsState &x : s)
    for (int l = 0; l < p->levels; l++) x.epoch[l] = updates;
  B2S_CUDA_CHECK(cudaMemcpy(p->d_state, s.data(), sizeof(HsState) * (size_t)p->batch, cudaMemcpyHostToDevice));
  p->host_updates = updates;
  return B2S_OK;
}

}  // extern "C"
