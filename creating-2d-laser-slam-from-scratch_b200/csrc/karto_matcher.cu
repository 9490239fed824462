// K1 — Karto correlative scan matcher on H100 (sm_90a).  Product code: CUDA only, no CPU fallback.
//
// Reference behaviour (paths relative to reference/lesson6/lib/open_karto):
//   ScanMatcher::Create / MatchScan / CorrelateScan / GetResponse / AddScans / FindValidPoints  src/Mapper.cpp:126-856
//   CorrelationGrid (smear kernel, ROI)                                   include/open_karto/Mapper.h:900-1118
//   GridIndexLookup::ComputeOffsets, Grid<T>, CoordinateConverter          include/open_karto/Karto.h:6409-6501, 4209-4767
//   LocalizedRangeScan::Update (point readings)                            include/open_karto/Karto.h:5362-5428
//
// Data layout in HBM (per handle, B = batch capacity, N = beams):
//   grids   [B][grid_pitch] u8      one correlation grid per match, same flat row-major layout as the reference
//                                   (index = x + y*width_step); grid_pitch = data_size rounded up to 128 B (+pad, zero)
//   lut     [B][nA][N]      i32     per-angle flat offsets (GridIndexLookup), INT32_MAX = INVALID_SCAN
//   sums    [B][nA][nY][nX] i32     integer numerators of GetResponse for the whole (x,y,theta) volume
//   probs   [B][side*side]  f64     per-cell maximum over theta (m_pSearchSpaceProbs)
//
// Kernels:
//   k_scan_points      point readings + scan-local points                              (fp64, O(B*N))
//   k_grid_offsets     grid offset that centres the ROI on the scan's sensor position
//   k_add_scan         FindValidPoints state machine + rasterise + max-smear           (byte atomics, O(B*S*N))
//   k_add_scans_seq    the same, sequential, when an off-centre smear value reaches 100 (order-dependent) or a base
//                      scan does not fit in k_add_scan's shared memory
//   k_grid_sat         per-match summed-area table of the grid's non-empty 4x4 blocks
//   k_grid_pool        per-match 4x4 and 7x7 max-pooled grids of the angle-pruning bound
//   k_bases            candidate lattice -> flat base indices; flags irregular and out-of-grid lattices
//   k_offsets          per-angle lookup tables                                         (fp64 -> i32)
//   k_offsets_sorted   window kernel's lists: window origins grouped by row band, byte alignment and interior /
//                      edge, empty windows dropped through the summed-area table (a pruned sweep: only the angles it
//                      sweeps)
//   k_sweep_window     THE HOT KERNEL: grid (or a row band of it) staged into shared memory by TMA bulk copy;
//                      one warp per (angle, 32x32 candidate tile), one lane per candidate row; each 32-bit
//                      shared-memory word feeds 4 adjacent-x candidates (byte-permute into packed u16
//                      accumulators)                                                    (int, issue bound)
//   k_sweep_bound (groups, probe, select), k_prune_select, k_count_empty
//                      angle pruning: an upper bound of every angle's responses from the pooled grid, an exact probe
//                      of the most promising angles, then k_sweep_window on only the angles that can matter
//   k_sweep_generic    any lattice / any grid size: one warp per (x,y) candidate, lanes over beams,
//                      gathers from global memory through L1/L2
//   k_reduce           penalties, best response, tie-averaged pose, positional covariance (fp64, one CTA per match);
//                      the whole tail or one phase of an angle-split sweep
//   k_angular_cov      fine-stage angular covariance (re-evaluates GetResponse at the best cell)
//   k_results_to_centers, k_status_pack, k_status_apply: small copies between the stages
//
// Which sweep kernel runs, with which band geometry and shared-memory sizes, is decided by plan_sweep
// (karto_sweep_plan.cuh) before anything is enqueued.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <type_traits>
#include <vector>

#include <math_constants.h>

#include "common.cuh"
#include "karto_sweep_plan.cuh"
#include "nccl_dl.cuh"
#include "scan_kernels.cuh"

namespace b2s {

// ----------------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------------

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// PRMT, default mode: selector nibble bit 3 replicates the sign bit of the selected byte.  Grid bytes are
// <= 100 < 128, so a "sign-replicated" byte is 0x00: one PRMT extracts two bytes into packed u16 lanes.
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}

// per-byte atomic max on a u8 array (no native byte atomics): CAS on the containing aligned word
// returns the byte's previous value
__device__ __forceinline__ uint32_t atomic_max_u8(uint8_t *base, int idx, uint32_t val) {
  uint32_t *w = reinterpret_cast<uint32_t *>(base + (idx & ~3));
  uint32_t shift = (idx & 3) * 8;
  uint32_t v = val << shift;
  uint32_t old = *w, assumed;
  do {
    if (((old >> shift) & 0xffu) >= val) return (old >> shift) & 0xffu;
    assumed = old;
    old = atomicCAS(w, assumed, __vmaxu4(assumed, v));
  } while (assumed != old);
  return (old >> shift) & 0xffu;
}

// ----------------------------------------------------------------------------------------------
// handle
// ----------------------------------------------------------------------------------------------

struct SweepDims {
  int nx = 0, ny = 0, na = 0;
};

}  // namespace b2s

using namespace b2s;

struct b2s_matcher {
  Stream stream;
  b2s_matcher_params p;
  b2s_laser l;
  b2s_grid_info g;
  int device = 0;
  int max_batch = 0, max_base = 0;
  int batch = 0, n = 0, n_base = 0;
  bool scans_set = false, grids_set = false;
  bool smear_degenerate = false;  // an off-centre kernel value reaches 100: AddScan becomes order-dependent
  size_t grid_pitch = 0;
  int force_kernel = 0;
  int num_sms = 1;  // the device's, set at create
  int smem_optin = 0;
  size_t win_static_smem = 0;  // k_sweep_window's static shared memory: comes out of the opt-in budget of its image
  size_t add_static_smem = 0;  // k_add_scan's, likewise for the base scan it stages

  Buf<uint8_t> d_kernel;
  Buf<double> d_ranges, d_poses, d_sensor, d_pts, d_local;
  Buf<uint8_t> d_grids;
  Buf<double> d_grid_off;
  Buf<double> d_base_ranges, d_base_poses, d_base_pts;
  Buf<double> d_pool;              // scan pool: readings of scans that serve as base scans again and again
  size_t pool_count = 0;
  Buf<int32_t> d_base_src;         // [batch * n_base] pool rows of the current base sets
  Buf<int32_t> d_lut;
  Buf<int32_t> d_lists, d_counts, d_starts;  // window kernel: per-(match, angle) grouped window origins
  Buf<double> d_part_best, d_glob_best, d_tie;  // split-sweep phases: [B], [B], [B][5]
  Buf<int32_t> d_status;                        // [B] statuses of a split sweep
  Event ev_split[6];
  double last_split_ms[4] = {0, 0, 0, 0};
  int last_k_first = 0;
  Buf<uint16_t> d_sat;  // [B][(sby+1)(sbx+1)] block summed-area tables of the grids
  int sbx = 0, sby = 0;
  bool sat_valid = false;
  Buf<unsigned long long> d_stats;      // [0] beam-angle pairs dropped as empty windows, [1] angles pruned, last sweep
  HostBuf<unsigned long long> h_stats;  // pinned copy, read back with the results
  PoolLayout pool[2];                   // the 4x4 and 7x7 max-pooled grids' layouts (pool_layout), fixed at create
  Buf<uint8_t> d_pools[2];              // [B][pool[i].pitch] the pooled grids (k_grid_pool), when they fit
  Buf<double> d_ubr;                    // [B][nA] angle bounds of a pruned sweep (NaN: not bounded one by one)
  Buf<double> d_gub;                    // [B][ceil(nA / BOUND_GROUP)] group bounds of a pruned sweep
  Buf<int32_t> d_n_eval;                // [B] angles k_prune_select left for k_sweep_bound<BOUND_SELECT>
  Buf<double> d_cuts;                   // [B] the pruning cut L - 0.1 - 1e-9 of each match
  Buf<int32_t> d_bscratch;              // [B][nA + groups] k_sweep_bound's angle lists and group order
  Buf<int32_t> d_angles, d_n_angles;    // [B][nA], [B]: the angle lists of a pruned sweep's two exact passes
  Buf<uint8_t> d_keep;                  // [B][nA] angles a pruned sweep swept
  SweepPlan last_plan;                  // of the last sweep
  bool last_pruned = false;             // the last sweep skipped angles: get_response_sums sweeps them first
  int last_batch = 0;                   // matches of the last sweep
  double last_pruned_frac = 0.0;
  bool pending = false;                   // a correlate_scan_begin awaits its _end
  int pending_batch = 0;                  // batch size that _begin enqueued
  double last_empty_frac = 0.0;
  bool empty_pending = false;  // the last sweep was pruned: its empty windows are counted when last_stats asks
  bool grid_high_bytes = false;  // set_grids saw a byte > 127: the packed-byte window kernel is not applicable
  Buf<int32_t> d_sums;
  Buf<int32_t> d_bases;  // [B][ny*nx] candidate base indices
  Buf<int32_t> d_flags;  // [B] per-match: bit0 lattice regular stride-1, bits 8.. status
  Buf<double> d_probs;
  Buf<double> d_centers;
  Buf<b2s_match_result> d_results;
  HostBuf<b2s_match_result> h_results;  // pinned
  Buf<int> d_work;                       // persistent-CTA work counter
  SweepDims last;
  b2s_search last_search;
  bool have_sweep = false;
  Event ev[4];
  double last_ms[4] = {0, 0, 0, 0};
  int last_path = 0;
};

namespace b2s {

// MatchScan steps 2-4 (Mapper.cpp:212-220): grid offset so that the ROI centre is the scan's sensor position
__global__ void k_grid_offsets(const double *__restrict__ sensor, double *__restrict__ grid_off, int batch, int roi_w,
                               int roi_h, double resolution) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  grid_off[2 * b] = sensor[3 * b] - (0.5 * (double)(roi_w - 1) * resolution);
  grid_off[2 * b + 1] = sensor[3 * b + 1] - (0.5 * (double)(roi_h - 1) * resolution);
}

// ----------------------------------------------------------------------------------------------
// k_add_scan: ScanMatcher::AddScan (Mapper.cpp:716-748) for one (match, base scan) per block:
// the FindValidPoints state machine (Mapper.cpp:756-811) runs over points staged in shared memory (see below),
// then all threads rasterise the valid points and max-stamp the smear kernel (Mapper.h:971-1005).
// The result is a per-byte maximum, hence independent of the order in which points / scans are applied,
// EXCEPT when an off-centre kernel value equals 100 (sigma ~ 10*res); that case takes k_add_scans_seq.
// ----------------------------------------------------------------------------------------------
// The state machine in parallel.  Its only carried state is the "first point of the current segment" f and the
// trailing index, and after every segment boundary (a point farther than 0.1 m from f) trailing == that boundary's
// index whichever branch ran.  Hence: (1) next[i] = first j > i with |p_i - p_j|^2 > 0.01 (same expression, so NaN /
// inf readings behave as in the loop) is computed for all i at once; (2) one thread follows f -> next[f] from the first
// non-NaN point — a chain of ~n/5 dependent shared-memory loads instead of n iterations of fp64 arithmetic; (3) for
// boundary k (f = b[k-1], c = b[k]) the side test is evaluated in parallel and the points [b[k-1]', b[k]) — from index 0
// for the first boundary — are valid iff ss >= 0 (i.e. !(ss < 0), NaN included).  Points after the last boundary are
// never pushed (the reference drops the tail, SURVEY.md §8 a3).  Bit-identical flags to the sequential loop (kept verbatim in k_add_scans_seq).
__global__ void k_add_scan(const double *__restrict__ base_pts, const double *__restrict__ sensor,
                           const double *__restrict__ grid_off, uint8_t *__restrict__ grids, size_t grid_pitch,
                           const uint8_t *__restrict__ kernel, b2s_grid_info g, double scale, int n, int n_base) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double *px = reinterpret_cast<double *>(smem_raw);
  double *py = px + n;
  int *nxt = reinterpret_cast<int *>(py + n);  // next[i]; reused as the boundary list b[k]
  int *bnd = nxt + n;
  uint8_t *valid = reinterpret_cast<uint8_t *>(bnd + n + 1);
  __shared__ int n_bnd, first_pt;
  const int bs = blockIdx.x;  // b * n_base + s
  const int b = bs / n_base;
  if (threadIdx.x == 0) first_pt = n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    px[i] = base_pts[((size_t)bs * n + i) * 2];
    py[i] = base_pts[((size_t)bs * n + i) * 2 + 1];
    valid[i] = 0;
  }
  __syncthreads();
  const double min_sq = 0.1 * 0.1;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double fx = px[i], fy = py[i];
    if (!isnan(fx) && !isnan(fy)) atomicMin(&first_pt, i);
    int j = i + 1;
    for (; j < n; j++) {
      const double dx = fx - px[j], dy = fy - py[j];
      if (dx * dx + dy * dy > min_sq) break;
    }
    nxt[i] = j;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int k = 0;
    for (int f = first_pt; f < n; f = nxt[f]) bnd[k++] = f;
    n_bnd = k;
  }
  __syncthreads();
  const double vx = sensor[3 * b], vy = sensor[3 * b + 1];
  for (int k = 1 + threadIdx.x; k < n_bnd; k += blockDim.x) {
    const int f = bnd[k - 1], c = bnd[k];
    const double fx = px[f], fy = py[f], cx = px[c], cy = py[c];
    const double a = vy - fy;
    const double bb = fx - vx;
    const double cc = fy * vx - fx * vy;
    const double ss = cx * a + cy * bb + cc;
    if (!(ss < 0.0))
      for (int t = (k == 1 ? 0 : f); t < c; t++) valid[t] = 1;
  }
  __syncthreads();
  // Rasterise + smear.  The result is max over occupied cells of the kernel stamped around them, and a cell holds 100
  // only as the centre of some point (no off-centre kernel value reaches 100 on this path), so each occupied cell is
  // stamped ONCE, by whichever thread raises its centre byte to 100 (running-window base scans hit the same walls many
  // times over).  Winners are queued in shared memory and stamped a warp at a time, lanes over the kernel cells.
  const double ox = grid_off[2 * b], oy = grid_off[2 * b + 1];
  uint8_t *grid = grids + (size_t)b * grid_pitch;
  const int half = g.kernel_size / 2;
  int *win = nxt;  // the chain arrays are free again
  if (threadIdx.x == 0) n_bnd = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!valid[i]) continue;
    double gxd = kround((px[i] - ox) * scale);
    double gyd = kround((py[i] - oy) * scale);
    // IsUpTo on static_cast<int>: non-finite / out-of-int-range values are rejected (see SURVEY.md §8 a3)
    if (!(gxd >= 0.0 && gxd < (double)g.roi_w) || !(gyd >= 0.0 && gyd < (double)g.roi_h)) continue;
    const int idx = ((int)gxd + g.roi_x) + ((int)gyd + g.roi_y) * g.width_step;
    if (atomic_max_u8(grid, idx, GRID_OCCUPIED) != GRID_OCCUPIED) win[atomicAdd(&n_bnd, 1)] = idx;
  }
  __syncthreads();
  // one lane per aligned 32-bit WORD of the stamp (a kernel row covers <= kernel_size/4 + 2 words): the four byte
  // maxima of a word go out as one packed CAS, so lanes of a warp never contend with each other
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, n_win = n_bnd;
  const int ks = g.kernel_size, wpr = (ks + 3) / 4 + 1;  // words per kernel row, whatever the alignment
  for (int w = warp; w < n_win; w += nwarps) {
    const int idx = win[w];
    for (int t = lane; t < ks * wpr; t += 32) {
      const int j = t / wpr - half, q = t % wpr;
      const int row0 = idx - half + j * g.width_step;   // byte index of the stamp row's first cell
      const int wbase = (row0 & ~3) + 4 * q;            // this lane's aligned word
      uint32_t v = 0;
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int k = wbase + e - row0;                 // kernel column of byte e
        if (k >= 0 && k < ks) v |= (uint32_t)kernel[k + ks * (j + half)] << (8 * e);
      }
      if (v == 0) continue;
      uint32_t *wp = reinterpret_cast<uint32_t *>(grid + wbase);
      uint32_t old = *wp, assumed;
      do {
        const uint32_t mx = __vmaxu4(old, v);
        if (mx == old) break;
        assumed = old;
        old = atomicCAS(wp, assumed, mx);
      } while (assumed != old);
    }
  }
}

// exact sequential AddScans for the degenerate smear kernel (see above): one thread per match
__global__ void k_add_scans_seq(const double *__restrict__ base_pts, const double *__restrict__ sensor,
                                const double *__restrict__ grid_off, uint8_t *__restrict__ grids, size_t grid_pitch,
                                const uint8_t *__restrict__ kernel, b2s_grid_info g, double scale, int n, int n_base,
                                int batch, uint8_t *__restrict__ valid_scratch) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  uint8_t *grid = grids + (size_t)b * grid_pitch;
  uint8_t *valid = valid_scratch + (size_t)b * n;
  const int half = g.kernel_size / 2;
  for (int s = 0; s < n_base; s++) {
    const double *p = base_pts + ((size_t)(b * n_base + s) * n) * 2;
    // FindValidPoints on strided xy pairs
    const double min_sq = 0.1 * 0.1;
    const double vx = sensor[3 * b], vy = sensor[3 * b + 1];
    for (int i = 0; i < n; i++) valid[i] = 0;
    int trailing = 0;
    double fx = 0.0, fy = 0.0;
    bool first_time = true;
    for (int it = 0; it < n; it++) {
      double cx = p[2 * it], cy = p[2 * it + 1];
      if (first_time && !isnan(cx) && !isnan(cy)) { fx = cx; fy = cy; first_time = false; }
      double dx = fx - cx, dy = fy - cy;
      if (dx * dx + dy * dy > min_sq) {
        double a = vy - fy, bb = fx - vx, c = fy * vx - fx * vy;
        double ss = cx * a + cy * bb + c;
        fx = cx; fy = cy;
        if (ss < 0.0) trailing = it;
        else for (; trailing != it; ++trailing) valid[trailing] = 1;
      }
    }
    for (int i = 0; i < n; i++) {
      if (!valid[i]) continue;
      double gxd = kround((p[2 * i] - grid_off[2 * b]) * scale);
      double gyd = kround((p[2 * i + 1] - grid_off[2 * b + 1]) * scale);
      if (!(gxd >= 0.0 && gxd < (double)g.roi_w) || !(gyd >= 0.0 && gyd < (double)g.roi_h)) continue;
      int gx = (int)gxd + g.roi_x, gy = (int)gyd + g.roi_y;
      int idx = gx + gy * g.width_step;
      if (grid[idx] == GRID_OCCUPIED) continue;  // Mapper.cpp:734-738
      grid[idx] = GRID_OCCUPIED;
      for (int j = -half; j <= half; j++)
        for (int k = -half; k <= half; k++) {
          uint8_t kv = kernel[(k + half) + g.kernel_size * (j + half)];
          uint8_t *c = grid + (gx + k) + (gy + j) * g.width_step;
          if (kv > *c) *c = kv;
        }
    }
  }
}

// GridIndexLookup::ComputeOffsets for one reading (Karto.h:6474-6499)
__device__ __forceinline__ int32_t lut_value(double r, double lx, double ly, double cosine, double sine, double gox,
                                             double goy, double scale, int width_step) {
  if (isnan(r) || isinf(r)) return INVALID_SCAN;
  double ox = __dsub_rn(__dmul_rn(cosine, lx), __dmul_rn(sine, ly));
  double oy = __dadd_rn(__dmul_rn(sine, lx), __dmul_rn(cosine, ly));
  // WorldToGrid(offset + rGridOffset): ((o + off) - off) * scale (Karto.h:6491, 4239-4251)
  int32_t gx = cast_i32(kround(__dmul_rn(__dsub_rn(__dadd_rn(ox, gox), gox), scale)));
  int32_t gy = cast_i32(kround(__dmul_rn(__dsub_rn(__dadd_rn(oy, goy), goy), scale)));
  return (int32_t)((uint32_t)gx + (uint32_t)gy * (uint32_t)width_step);  // Grid<T>::GridIndex, no ROI
}

// ----------------------------------------------------------------------------------------------
// k_offsets: GridIndexLookup::ComputeOffsets (Karto.h:6455-6501).  One block per (match, angle).
// ----------------------------------------------------------------------------------------------
__global__ void k_offsets(const double *__restrict__ ranges, const double *__restrict__ local,
                          const double *__restrict__ grid_off, const double *__restrict__ centers, int center_stride,
                          double angle_center_override, int use_override, double angle_offset, double angle_res,
                          int n_angles, int n, int width_step, double scale, int32_t *__restrict__ lut, int k_first) {
  const int b = blockIdx.x / n_angles, k = blockIdx.x % n_angles;
  const double center = use_override ? angle_center_override : centers[(size_t)b * center_stride + 2];
  const double start = center - angle_offset;
  const double angle = start + (double)(uint32_t)(k_first + k) * angle_res;  // k_first: angle subset of a split sweep
  const double cosine = cos(angle), sine = sin(angle);
  const double gox = grid_off[2 * b], goy = grid_off[2 * b + 1];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int32_t v = lut_value(ranges[(size_t)b * n + i], local[((size_t)b * n + i) * 2], local[((size_t)b * n + i) * 2 + 1],
                                cosine, sine, gox, goy, scale, width_step);
    lut[((size_t)b * n_angles + k) * n + i] = v;
  }
}

// ----------------------------------------------------------------------------------------------
// k_bases: candidate lattice of CorrelateScan (Mapper.cpp:338-358, 373-386) -> flat base index per (iy, ix).
// flags[b]: bit0 = lattice is the regular raster base00 + stride*(ix + iy*width_step), stride = 1 or 2 cells;
//           bit1 = some candidate fell outside the grid (reference throws karto::Exception, Karto.h:4490-4499)
// ----------------------------------------------------------------------------------------------
__global__ void k_bases(const double *__restrict__ centers, const double *__restrict__ grid_off, b2s_search s,
                        b2s_grid_info g, double scale, int nx, int ny, int32_t *__restrict__ bases,
                        int32_t *__restrict__ flags, int stride) {
  const int b = blockIdx.x;
  __shared__ int irregular, oob;
  if (threadIdx.x == 0) { irregular = 0; oob = 0; }
  __syncthreads();
  const double cx = centers[3 * b], cy = centers[3 * b + 1];
  const double gox = grid_off[2 * b], goy = grid_off[2 * b + 1];
  const double start_x = -s.offset_x, start_y = -s.offset_y;
  const int32_t gx0 = world_to_grid_1(cx + start_x, gox, scale) + g.roi_x;
  const int32_t gy0 = world_to_grid_1(cy + start_y, goy, scale) + g.roi_y;
  for (int c = threadIdx.x; c < nx * ny; c += blockDim.x) {
    int iy = c / nx, ix = c % nx;
    double y = start_y + (double)(uint32_t)iy * s.res_y;
    double x = start_x + (double)(uint32_t)ix * s.res_x;
    int32_t gx = world_to_grid_1(cx + x, gox, scale) + g.roi_x;  // CorrelationGrid::GridIndex (Mapper.h:941-947)
    int32_t gy = world_to_grid_1(cy + y, goy, scale) + g.roi_y;
    if (!(gx >= 0 && gx < g.width && gy >= 0 && gy < g.height)) oob = 1;
    if (gx != gx0 + stride * ix || gy != gy0 + stride * iy) irregular = 1;
    bases[(size_t)b * nx * ny + c] = gx + gy * g.width_step;
  }
  __syncthreads();
  if (threadIdx.x == 0) flags[b] = (irregular ? 0 : 1) | (oob ? 2 : 0);
}

// ----------------------------------------------------------------------------------------------
// k_sweep_generic: integer numerators of GetResponse (Mapper.cpp:819-856) for every candidate.
// One warp per (x,y) candidate, looping over all angles; lanes stride over beams; grid + LUT read from
// global memory (L1/L2).  Handles any lattice and any grid size.  mode 0: all matches; mode 1: only matches
// whose lattice is NOT regular (the window kernel did the others).
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sweep_generic(const uint8_t *__restrict__ grids, size_t grid_pitch,
                                                       int data_size, const int32_t *__restrict__ lut,
                                                       const int32_t *__restrict__ bases,
                                                       const int32_t *__restrict__ flags, int mode, int n, int na,
                                                       int ncell, int32_t *__restrict__ sums,
                                                       const double *__restrict__ ranges,
                                                       const double *__restrict__ local,
                                                       const double *__restrict__ grid_off,
                                                       const double *__restrict__ centers, double angle_offset,
                                                       double angle_res, int width_step, double scale, int k_first,
                                                       int batch) {
  for (int b = blockIdx.y; b < batch; b += gridDim.y) {
    const int f = flags[b];
    if (f & 2) continue;
    if (mode == 1 && (f & 1)) continue;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint8_t *grid = grids + (size_t)b * grid_pitch;
    for (int c = blockIdx.x * (blockDim.x >> 5) + warp; c < ncell; c += gridDim.x * (blockDim.x >> 5)) {
      const int32_t base = bases[(size_t)b * ncell + c];
      for (int k = 0; k < na; k++) {
        const int32_t *offs = lut ? lut + ((size_t)b * na + k) * n : nullptr;
        double cosine = 0, sine = 0, gox = 0, goy = 0;
        if (!lut) {  // no materialised table (window mode fall-through): GridIndexLookup values on the fly
          const double angle = (centers[(size_t)b * 3 + 2] - angle_offset) + (double)(uint32_t)(k_first + k) * angle_res;
          cosine = cos(angle); sine = sin(angle);
          gox = grid_off[2 * b]; goy = grid_off[2 * b + 1];
        }
        int32_t sum = 0;
        if (lut) {
          // 8 independent (offset, cell) load chains in flight per lane: the gather is latency bound
          constexpr int U = 8;
          for (int i0 = lane; i0 < n; i0 += 32 * U) {
            int32_t o[U];
#pragma unroll
            for (int u = 0; u < U; u++) o[u] = (i0 + 32 * u < n) ? __ldg(offs + i0 + 32 * u) : INVALID_SCAN;
            uint32_t v[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
              const int32_t idx = (int32_t)((uint32_t)base + (uint32_t)o[u]);
              v[u] = (o[u] != INVALID_SCAN && idx >= 0 && idx < data_size) ? (uint32_t)__ldg(grid + idx) : 0u;
            }
#pragma unroll
            for (int u = 0; u < U; u++) sum += (int32_t)v[u];
          }
        } else {
          for (int i = lane; i < n; i += 32) {
            const int32_t o = lut_value(ranges[(size_t)b * n + i], local[((size_t)b * n + i) * 2],
                                        local[((size_t)b * n + i) * 2 + 1], cosine, sine, gox, goy, scale, width_step);
            if (o == INVALID_SCAN) continue;
            const int32_t idx = (int32_t)((uint32_t)base + (uint32_t)o);
            if (idx >= 0 && idx < data_size) sum += __ldg(grid + idx);
          }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
        if (lane == 0) sums[((size_t)b * na + k) * ncell + c] = sum;
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// k_sweep_window — the hot kernel (stride-1 lattices, grid fits in shared memory).
//
// For a fixed angle k and beam i, the cells read by all (ix, iy) candidates form the nY x nX window of the
// grid whose origin is  a = base00 + lut[k][i]  (flat index; rows are width_step apart).  So
//     sums[k][iy][ix] = SUM_i grid[a_i + iy*width_step + ix].
// A persistent CTA stages one match's whole grid into shared memory with TMA bulk copies and its warps take
// (angle, 32x32 window tile) work items.  Within a warp lane r owns candidate row r.
//
// k_offsets_sorted prepares, per (match, angle), the window origins a_i grouped by byte alignment (a & 3) and
// split into INTERIOR beams (every byte any lane will touch lies inside the staged image, no checks needed) and
// EDGE beams (some row leaves [0, data_size): per-row redirect to a zero guard), with beams whose whole window is
// outside dropped.  Integer sums commute, so the regrouping is free.
//
// Inner loop, per PAIR of same-alignment beams and per lane: 2 x 9 aligned 32-bit shared-memory loads (the 36
// bytes covering the lane's 32 candidate cells), 9 packed-byte adds of the two beams' words (cell values <= 100,
// so two fit a byte), then each summed word is added whole to one accumulator and its bytes 1,3 (one byte permute) to
// a packed-u16 one; bytes 0,2 are recovered as the difference at the flush, so they need no mask per word.  The 18
// accumulators are kept in WORD-ALIGNED coordinates — the alignment (a compile-time constant of the class) is only
// applied when the u16 lanes are flushed into the 32 per-candidate 32-bit sums.  The sweep is bound by instruction
// issue (DESIGN.md §4): one shared-memory word feeds 4 adjacent-x candidates for ~2 integer instructions per beam.
//
// Flat-index semantics of the reference are kept bit-exactly: rows wrap exactly as `base + offset` does, and
// positions outside [0, data_size) read zeros (guard bands, zero padding of the HBM image, redirect of rows that
// are entirely outside).  Lanes 16..31 fetch their 9 words rotated by one so that the two half-warps hit odd /
// even banks (width_step/4 is even, so rows r and r+16 would otherwise always collide).
// ----------------------------------------------------------------------------------------------
// (WIN_THREADS, WIN_GUARD, WIN_MAX_BANDS, LIST_PAD: karto_sweep_plan.cuh)
constexpr int WIN_FLUSH_BEAMS = 512;    // beams accumulated in u16 lanes between flushes (512 * 127 < 65536)
constexpr int32_t WIN_SKIP = -(1 << 29);

// ----------------------------------------------------------------------------------------------
// k_grid_sat: per match, a summed-area table over 4x4-cell blocks of "block holds a non-zero cell".  A beam whose
// whole nY x nX window covers only empty blocks adds 0 to every candidate, so k_offsets_sorted may drop it — the
// response volume stays bit-identical.  sat[(by+1) x (bx+1)] u16, one block per match.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_grid_sat(const uint8_t *__restrict__ grids, size_t grid_pitch, int width_step, int height, int bx, int by,
               uint16_t *__restrict__ sat_all) {
  extern __shared__ uint32_t s_sat[];  // (by+1) x (bx+1)
  const int b = blockIdx.x;
  const uint8_t *grid = grids + (size_t)b * grid_pitch;
  const int W = bx + 1;
  for (int i = threadIdx.x; i < (by + 1) * W; i += blockDim.x) s_sat[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < bx * by; i += blockDim.x) {
    const int cy = i / bx, cx = i % bx;
    uint32_t any = 0;
    for (int r = 0; r < 4; r++) {
      const int y = cy * 4 + r;
      if (y < height) any |= *reinterpret_cast<const uint32_t *>(grid + (size_t)y * width_step + cx * 4);  // width_step % 4 == 0
    }
    s_sat[(cy + 1) * W + (cx + 1)] = any ? 1u : 0u;
  }
  __syncthreads();
  for (int y = threadIdx.x + 1; y <= by; y += blockDim.x) {  // row prefix sums
    uint32_t acc = 0;
    for (int x = 1; x <= bx; x++) { acc += s_sat[y * W + x]; s_sat[y * W + x] = acc; }
  }
  __syncthreads();
  for (int x = threadIdx.x + 1; x <= bx; x += blockDim.x) {  // column prefix sums
    uint32_t acc = 0;
    for (int y = 1; y <= by; y++) { acc += s_sat[y * W + x]; s_sat[y * W + x] = acc; }
  }
  __syncthreads();
  uint16_t *out = sat_all + (size_t)b * (size_t)(((by + 1) * W + 7) & ~7);  // padded stride: k_offsets_sorted copies 16 bytes at a time
  for (int i = threadIdx.x; i < (by + 1) * W; i += blockDim.x) out[i] = (uint16_t)s_sat[i];  // < 65536 blocks (checked by the host)
}

// ----------------------------------------------------------------------------------------------
// k_grid_pool<K>: per match, the K x K max-pooled grid (K = 4: P of k_sweep_bound; K = 7: P7 of k_sweep_bound_group)
// in its four residue planes (layout: pool_layout and pool_index in
// karto_sweep_plan.cuh).  The pooling is in FLAT index space, rows wrapping exactly as a candidate's `base + offset`
// does, so the pooled byte at a block's corner is at least every byte a candidate of that block reads.  Thread q pools
// P[f] for the 16 indices j = f + lead in [16q, 16q + 16) and writes word q of each plane; grid bytes outside
// [0, data_size) count as 0, so the planes' padding comes out 0.
// grid(ceil(plane / 1024), B), 256 threads.
// ----------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256)
    k_grid_pool(const uint8_t *__restrict__ grids, size_t grid_pitch, int data_size, int width_step,
                int lead, int plane, uint8_t *__restrict__ pools, size_t pitch, int batch) {
  static_assert(K == 4 || K == 7, "4x4 or 7x7 pooling");
  constexpr int NW = K == 4 ? 5 : 6;  // words per row: the 16 positions and the K - 1 bytes after them
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q * 4 >= plane) return;
  for (int b = blockIdx.y; b < batch; b += gridDim.y) {
    const uint8_t *grid = grids + (size_t)b * grid_pitch;
    const int f = 16 * q - lead;  // a multiple of 4, as are width_step and data_size
    auto word = [&](int r) { return (r >= 0 && r < data_size) ? __ldg(reinterpret_cast<const uint32_t *>(grid + r)) : 0u; };
    uint32_t m[4] = {0, 0, 0, 0};  // byte r of m[t] = P[f + 4t + r]
#pragma unroll
    for (int dy = 0; dy < K; dy++) {
      const int r = f + dy * width_step;
      uint32_t w[NW];
#pragma unroll
      for (int t = 0; t < NW; t++) w[t] = word(r + 4 * t);
      uint32_t m4[NW - 1];  // byte i of m4[t] = max of row bytes 4t + i .. 4t + i + 3
#pragma unroll
      for (int t = 0; t < NW - 1; t++) {
        const uint32_t a = __vmaxu4(w[t], __funnelshift_r(w[t], w[t + 1], 8));
        const uint32_t c = __vmaxu4(__funnelshift_r(w[t], w[t + 1], 16), __funnelshift_r(w[t], w[t + 1], 24));
        m4[t] = __vmaxu4(a, c);
      }
#pragma unroll
      for (int t = 0; t < 4; t++)  // K = 7: bytes i .. i + 6 = bytes i .. i + 3 and i + 3 .. i + 6
        m[t] = __vmaxu4(m[t], K == 4 ? m4[t] : __vmaxu4(m4[t], __funnelshift_r(m4[t], m4[t + (K == 4 ? 0 : 1)], 24)));
    }
    // 4 x 4 byte transpose: plane r word q = byte r of m[0..3]
    const uint32_t lo01 = __byte_perm(m[0], m[1], 0x5140), hi01 = __byte_perm(m[0], m[1], 0x7362);
    const uint32_t lo23 = __byte_perm(m[2], m[3], 0x5140), hi23 = __byte_perm(m[2], m[3], 0x7362);
    uint8_t *out = pools + (size_t)b * pitch + 4 * q;
    *reinterpret_cast<uint32_t *>(out) = __byte_perm(lo01, lo23, 0x5410);
    *reinterpret_cast<uint32_t *>(out + plane) = __byte_perm(lo01, lo23, 0x7632);
    *reinterpret_cast<uint32_t *>(out + 2 * plane) = __byte_perm(hi01, hi23, 0x5410);
    *reinterpret_cast<uint32_t *>(out + 3 * plane) = __byte_perm(hi01, hi23, 0x7632);
  }
}

// ----------------------------------------------------------------------------------------------
// A beam's window origin and class at one angle: the one definition that k_offsets_sorted (which lists the beams) and
// k_sweep_bound (which bounds an angle from the same beams without lists) share, so that the two cannot disagree.
// ----------------------------------------------------------------------------------------------
// the angle k (counted from the search's first angle, k_first + index for an angle subset) of GridIndexLookup's table
__device__ __forceinline__ double win_angle(double center, double angle_offset, double angle_res, int k) {
  return (center - angle_offset) + (double)(uint32_t)k * angle_res;
}

// The geometry of one match's window lists (everything but the angle and the beam)
struct WinGeom {
  double gox, goy, scale;  // the grid offset of the match and 1 / resolution
  int32_t base00;          // flat index of candidate (0, 0)
  int32_t span32;          // last byte any lane may touch past a window origin, clamped to 2^29
  int width_step, data_size, height;
  int fx, fy;              // footprint of the candidate lattice in cells
  float inv_step, inv_band;
  int band_rows, nbands, neg_bands;
};

__device__ __forceinline__ WinGeom win_geom(double gox, double goy, double scale, int32_t base00, int stride,
                                            int rows_total, int cols_total, int width_step, int data_size, int height,
                                            int nx, int ny, int band_rows, int nbands, int neg_bands) {
  WinGeom G;
  G.gox = gox; G.goy = goy; G.scale = scale; G.base00 = base00;
  const long long span = (long long)stride * (rows_total - 1) * width_step + cols_total + 8;  // last byte any lane may touch
  G.span32 = (int32_t)min(span, (long long)(1 << 29));
  G.width_step = width_step; G.data_size = data_size; G.height = height;
  G.fx = stride * (nx - 1) + 1; G.fy = stride * (ny - 1) + 1;
  G.inv_step = 1.0f / (float)width_step; G.inv_band = 1.0f / (float)band_rows;
  G.band_rows = band_rows; G.nbands = nbands; G.neg_bands = neg_bands;
  return G;
}

// Scan-local point (plx, ply) at the angle with the given cosine and sine: `a` = the window origin (base00 + the
// GridIndexLookup value, flat index), returned = its group: 255 (dropped: the window lies wholly outside the grid, or
// the point is not finite, or - when use_sat - every 4x4 block the window covers is empty, which sets `empty`), else
// 8 * band + (a & 3) for an interior window, 8 * band + 4 + (a & 3) for an edge one.
__device__ __forceinline__ int win_origin_class(double plx, double ply, double cosine, double sine, const WinGeom &G,
                                                bool use_sat, const uint16_t *__restrict__ sat, int SW, int32_t &a,
                                                bool &empty) {
  // lut_value() inlined: a non-finite local point (INVALID_SCAN reading) makes ox/oy non-finite
  const double ox = __dsub_rn(__dmul_rn(cosine, plx), __dmul_rn(sine, ply));
  const double oy = __dadd_rn(__dmul_rn(sine, plx), __dmul_rn(cosine, ply));
  int cls = 255;  // dropped
  a = 0;
  empty = false;
  if (isfinite(ox) && isfinite(oy)) {
    const int32_t gx = cast_i32(kround(__dmul_rn(__dsub_rn(__dadd_rn(ox, G.gox), G.gox), G.scale)));
    const int32_t gy = cast_i32(kround(__dmul_rn(__dsub_rn(__dadd_rn(oy, G.goy), G.goy), G.scale)));
    const int32_t o = (int32_t)((uint32_t)gx + (uint32_t)gy * (uint32_t)G.width_step);
    a = (int32_t)((uint32_t)G.base00 + (uint32_t)o);
    // window [a - 8, a + span] against [0, data_size): 32-bit arithmetic after clamping far-away origins
    const int32_t ac = max(min(a, (int32_t)(1 << 29)), -(int32_t)(1 << 29));
    const int32_t lo = ac - 8, hi = ac + G.span32;
    if (hi < 0 || lo >= G.data_size) cls = 255;  // whole window outside: contributes 0
    else if (lo >= -(WIN_GUARD - 16) && hi <= G.data_size + (WIN_GUARD - 16)) cls = a & 3;  // interior
    else cls = 4 + (a & 3);                                                                  // edge
    int y = 0, x = 0;
    if ((use_sat || G.nbands > 1) && cls < 255 && (a >= 0 || G.neg_bands > 0)) {
      // floor(a / width_step) by float reciprocal + fix-up (|a| < 2^24 is exact in float; larger values are
      // corrected too); a < 0 only matters when origins below the grid get row bands of their own (neg_bands)
      if (G.data_size <= (1 << 24) && ac == a) {
        y = (int)((float)a * G.inv_step);
        if (y * G.width_step > a) y--;
        else if ((y + 1) * G.width_step <= a) y++;
      } else {
        y = a / G.width_step;
        if (y * G.width_step > a) y--;
      }
      x = a - y * G.width_step;
    }
    if (G.nbands > 1 && cls < 8) {
      int band = (int)((float)y * G.inv_band);
      if (band * G.band_rows > y) band--;
      else if ((band + 1) * G.band_rows <= y) band++;
      cls += 8 * max(min(band + G.neg_bands, G.nbands - 1), 0);  // the row band that holds the window origin
    }
    if (use_sat && cls < 255 && a >= 0) {
      // empty-window test on the 4x4-block summed-area table (only for windows that do not wrap a row end)
      if (x + G.fx <= G.width_step && y + G.fy <= G.height) {
        const int bx0 = x >> 2, bx1 = (x + G.fx - 1) >> 2, by0 = y >> 2, by1 = (y + G.fy - 1) >> 2;
        const uint32_t c = (uint32_t)sat[(by1 + 1) * SW + bx1 + 1] - (uint32_t)sat[by0 * SW + bx1 + 1] -
                           (uint32_t)sat[(by1 + 1) * SW + bx0] + (uint32_t)sat[by0 * SW + bx0];
        if (c == 0) { cls = 255; empty = true; }
      }
    }
  }
  return cls;
}

// One block per (match, chunk of OFF_CHUNK angles): window origins grouped as [I0 I1 I2 I3 E0 E1 E2 E3] (I = interior,
// E = edge, index = a & 3), every group a multiple of 4 long (an interior group donates its 0..3 surplus beams to its edge
// group; edge groups are padded with far-negative sentinels of the same alignment).  counts[8] holds the group lengths.
// The scan's readings and local points are staged in shared memory once per block and reused for every angle of
// the chunk (16x less L2 traffic than one block per angle).  A non-finite reading (INVALID_SCAN, Karto.h:6478) always
// yields a non-finite local point (inf/NaN propagate through the inverse transform), so only the points are staged.
// LISTED (a pruned sweep): the block lists the angles at positions [k0, k0 + OFF_CHUNK) of match b's angle list
// list_angles[b * n_angles ...] (list_n[b] long, list_chunks blocks per match), each at its own index k, so that
// k_sweep_window reads them where it reads every angle's lists; the lists of the other angles are left as they were.
// (OFF_CHUNK, OFF_Q, OFF_SMEM_PER_BEAM: karto_sweep_plan.cuh)
constexpr int OFF_GS = 8 * WIN_MAX_BANDS;             // group slots per angle
template <bool LISTED>
__global__ void __launch_bounds__(256)
    k_offsets_sorted(const double *__restrict__ ranges, const double *__restrict__ local,
                     const double *__restrict__ grid_off, const double *__restrict__ centers,
                     const int32_t *__restrict__ bases, const int32_t *__restrict__ flags, double angle_offset,
                     double angle_res, int n_angles, int n, int ncell, int width_step, int data_size, double scale,
                     int rows_total, int cols_total, int32_t *__restrict__ lists, int32_t *__restrict__ counts,
                     const uint16_t *__restrict__ sat_all, int sbx, int sby, int height, int nx, int ny,
                     unsigned long long *__restrict__ stats, int band_rows, int nbands,
                     int32_t *__restrict__ starts, int stride, int k_first, int neg_bands,
                     const int32_t *__restrict__ list_angles, const int32_t *__restrict__ list_n, int list_chunks) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  double *s_lx = reinterpret_cast<double *>(s_raw), *s_ly = s_lx + n;  // [n] scan-local points
  int32_t *s_vals = reinterpret_cast<int32_t *>(s_ly + n);             // [OFF_Q][n] window origins
  uint8_t *s_cls = reinterpret_cast<uint8_t *>(s_vals + OFF_Q * n);    // [OFF_Q][n] group ids
  uint16_t *s_sat = reinterpret_cast<uint16_t *>(s_raw + (((size_t)n * OFF_SMEM_PER_BEAM + 15) & ~(size_t)15));  // [(sby+1)(sbx+1)] or unused
  __shared__ int cnt[OFF_Q * OFF_GS], fill[OFF_Q * OFF_GS], seg[OFF_Q * OFF_GS];  // [angle][band][group]
  __shared__ int n_empty;
  const int ngroups = 8 * nbands;
  const int list_cap = n + LIST_PAD * nbands;
  const int chunks = LISTED ? list_chunks : (n_angles + OFF_CHUNK - 1) / OFF_CHUNK;
  const int b = blockIdx.x / chunks, k0 = (blockIdx.x % chunks) * OFF_CHUNK;
  const int f = flags[b];
  if ((f & 2) || !(f & 1)) return;  // error / irregular lattice: the generic kernel handles this match
  if (LISTED && k0 >= list_n[b]) return;  // past the end of the match's angle list
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s_lx[i] = local[((size_t)b * n + i) * 2];
    s_ly[i] = local[((size_t)b * n + i) * 2 + 1];
  }
  const int SW = sbx + 1;
  if (sat_all) {  // per-match tables are padded to a multiple of 8 entries: 16-byte copies
    const int sat_stride = ((sby + 1) * SW + 7) & ~7;
    const uint4 *src = reinterpret_cast<const uint4 *>(sat_all + (size_t)b * sat_stride);
    uint4 *dst = reinterpret_cast<uint4 *>(s_sat);
    for (int i = threadIdx.x; i < sat_stride / 8; i += blockDim.x) dst[i] = src[i];
  }
  if (threadIdx.x == 0) n_empty = 0;
  const double center = centers[(size_t)b * 3 + 2];
  __shared__ double s_cos[OFF_CHUNK], s_sin[OFF_CHUNK];
  __shared__ int s_k[LISTED ? OFF_CHUNK : 1];  // LISTED: the angle index of each list position of the chunk
  if (threadIdx.x < OFF_CHUNK && k0 + threadIdx.x < (LISTED ? list_n[b] : n_angles)) {  // one sincos per angle, not per thread
    int k = k0 + threadIdx.x;
    if (LISTED) s_k[threadIdx.x] = k = list_angles[(size_t)b * n_angles + k];
    const double ang = win_angle(center, angle_offset, angle_res, k_first + k);
    s_cos[threadIdx.x] = cos(ang);
    s_sin[threadIdx.x] = sin(ang);
  }
  const WinGeom G = win_geom(grid_off[2 * b], grid_off[2 * b + 1], scale, bases[(size_t)b * ncell], stride, rows_total,
                             cols_total, width_step, data_size, height, nx, ny, band_rows, nbands, neg_bands);
  const int kend = min(k0 + OFF_CHUNK, LISTED ? list_n[b] : n_angles);  // one past the chunk's last list position
  for (int kq = k0; kq < kend; kq += OFF_Q) {  // OFF_Q angles per pass: half the barriers, one read of the points
    const int nq = min(OFF_Q, kend - kq);
    __syncthreads();  // staging done / previous angles' smem fully consumed
    for (int t = threadIdx.x; t < OFF_Q * OFF_GS; t += blockDim.x) { cnt[t] = 0; fill[t] = 0; }
    __syncthreads();
    int empty_here = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double plx = s_lx[i], ply = s_ly[i];
#pragma unroll
      for (int q = 0; q < OFF_Q; q++) {
        if (q >= nq) break;
        int32_t a;
        bool empty;
        const int cls = win_origin_class(plx, ply, s_cos[kq - k0 + q], s_sin[kq - k0 + q], G, sat_all != nullptr, s_sat,
                                         SW, a, empty);
        empty_here += empty;
        s_vals[q * n + i] = a;
        s_cls[q * n + i] = (uint8_t)cls;
        if (cls < 255) atomicAdd(&cnt[q * OFF_GS + cls], 1);
      }
    }
    if (empty_here) atomicAdd(&n_empty, empty_here);
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < nq) {  // one thread (of its own warp) per angle
      int *c_ = cnt + (threadIdx.x >> 5) * OFF_GS, *seg_ = seg + (threadIdx.x >> 5) * OFF_GS;
      int pos = 0;
      for (int g8 = 0; g8 < ngroups; g8 += 8) {
        for (int c = 0; c < 4; c++) {
          const int d = c_[g8 + c] & 3;  // interior groups are multiples of 4: the last-placed 0..3 beams go to the edge group
          c_[g8 + c] -= d;
          c_[g8 + 4 + c] += d;
        }
        for (int c = 0; c < 8; c++) {
          seg_[g8 + c] = pos;
          pos += (c_[g8 + c] + 3) & ~3;
        }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
#pragma unroll
      for (int q = 0; q < OFF_Q; q++) {
        if (q >= nq) break;
        int cls = s_cls[q * n + i];
        if (cls == 255) continue;
        int slot = atomicAdd(&fill[q * OFF_GS + cls], 1);
        if ((cls & 7) < 4 && slot >= cnt[q * OFF_GS + cls]) {  // a donated one
          cls += 4;
          slot = atomicAdd(&fill[q * OFF_GS + cls], 1);
        }
        const int k = LISTED ? s_k[kq - k0 + q] : kq + q;
        lists[((size_t)b * n_angles + k) * list_cap + seg[q * OFF_GS + cls] + slot] = s_vals[q * n + i];
      }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nq * ngroups; t += blockDim.x) {
      const int q = t / ngroups, g = t % ngroups;
      const int cg = cnt[q * OFF_GS + g], sg_ = seg[q * OFF_GS + g];
      const int k = LISTED ? s_k[kq - k0 + q] : kq + q;
      int32_t *out = lists + ((size_t)b * n_angles + k) * list_cap;
      if ((g & 7) >= 4)
        for (int r = cg; r < ((cg + 3) & ~3); r++)
          out[sg_ + r] = WIN_SKIP + (g & 3);  // pad: all-outside beams of the same alignment
      counts[((size_t)b * n_angles + k) * ngroups + g] = (cg + 3) & ~3;
      starts[((size_t)b * n_angles + k) * ngroups + g] = sg_;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && stats && n_empty) atomicAdd(stats, (unsigned long long)n_empty);
}

// flush the packed-u16 accumulators (word-aligned coordinates, alignment class SH) into the per-candidate sums.
// slots 0..7 hold aligned word j (lanes 0..15) or aligned word (j+1)%8 (lanes 16..31); slot 8 holds aligned word 8;
// byte q of word w is candidate x = 4*w + q - SH.
// With STRIDE = 2 (candidates every other cell) only the bytes at even distance from the origin are candidates:
// byte position p = 4*w + q - SH is candidate x = p / 2 when p is even; a tile then holds 16 candidates in 32 bytes.
template <int SH, int STRIDE, int ROT>
__device__ __forceinline__ void win_flush_rot(const uint32_t (&lo)[9], const uint32_t (&hi)[9], uint32_t (&acc)[32]) {
#define B2S_FLUSH_ONE(P, VAL)                                                        \
  if ((P) >= 0 && ((P) % STRIDE) == 0 && (P) / STRIDE < 32 / STRIDE) acc[((P) / STRIDE) & 31] += (VAL);
#define B2S_FLUSH_SLOT(J, W)                                                         \
  {                                                                                  \
    const int x0 = 4 * (W) - SH;                                                     \
    B2S_FLUSH_ONE(x0 + 0, lo[J] & 0xffffu)                                           \
    B2S_FLUSH_ONE(x0 + 1, hi[J] & 0xffffu)                                           \
    B2S_FLUSH_ONE(x0 + 2, lo[J] >> 16)                                               \
    B2S_FLUSH_ONE(x0 + 3, hi[J] >> 16)                                               \
  }
#pragma unroll
  for (int j = 0; j < 8; j++) B2S_FLUSH_SLOT(j, (j + ROT) % 8)
  B2S_FLUSH_SLOT(8, 8)
#undef B2S_FLUSH_SLOT
#undef B2S_FLUSH_ONE
}

// `rot` = this lane's word rotation: slot j holds aligned word (j + rot) % 8 (see win_load).  GEN = false: rot is 0 for
// lanes 0..15 and 1 for lanes 16..31; GEN = true: any of 0..7.
template <int SH, int STRIDE, bool GEN>
__device__ __forceinline__ void win_flush(uint32_t (&lo)[9], uint32_t (&hi)[9], uint32_t (&acc)[32], int rot) {
  // lo holds the plain 32-bit sum of the packed words (see win_accumulate2); taking away bytes 1 and 3, which hi
  // holds as u16 lanes, leaves bytes 0 and 2 as u16 lanes.  Exact modulo 2^32 because every u16 lane is < 65536.
#pragma unroll
  for (int j = 0; j < 9; j++) lo[j] -= hi[j] << 8;
  if (!GEN) {
    if (!rot) win_flush_rot<SH, STRIDE, 0>(lo, hi, acc);
    else win_flush_rot<SH, STRIDE, 1>(lo, hi, acc);
  } else {
    switch (rot) {
      case 0: win_flush_rot<SH, STRIDE, 0>(lo, hi, acc); break;
      case 1: win_flush_rot<SH, STRIDE, 1>(lo, hi, acc); break;
      case 2: win_flush_rot<SH, STRIDE, 2>(lo, hi, acc); break;
      case 3: win_flush_rot<SH, STRIDE, 3>(lo, hi, acc); break;
      case 4: win_flush_rot<SH, STRIDE, 4>(lo, hi, acc); break;
      case 5: win_flush_rot<SH, STRIDE, 5>(lo, hi, acc); break;
      case 6: win_flush_rot<SH, STRIDE, 6>(lo, hi, acc); break;
      default: win_flush_rot<SH, STRIDE, 7>(lo, hi, acc); break;
    }
  }
#pragma unroll
  for (int j = 0; j < 9; j++) { lo[j] = 0; hi[j] = 0; }
}

// load the 8 (+1) words of one beam's row; `base` = byte address in sgrid of aligned word 0 of this lane's row.
// Bank conflicts: lane L's row starts (L * STRIDE * width_step / 4) mod 32 banks after lane 0's; with width_step a
// multiple of 8 that step is even, so m = gcd(step, 32) >= 2 lanes share every row-start bank.  Rotating the order in
// which a lane fetches its 8 words by rot = L / (32 / m) gives each of those m lanes a different bank at every load
// instruction, and the m-lane groups tile the 32 banks when m <= 8: conflict-free.  The common case m = 2 (cfg 1/2's
// 408-byte step: 102 words) is the GEN = false path, lanes 16..31 fetch words 1..7,0 with immediate offsets; GEN =
// true takes any rotation through per-lane byte offsets `loff`.  Word 8 (only needed when the window's last
// candidates spill past 32 bytes) cannot be de-conflicted and is loaded only when W9.
template <bool W9, bool GEN>
__device__ __forceinline__ void win_load(const uint8_t *__restrict__ sgrid, int base, int rot, const int (&loff)[8],
                                         uint32_t (&v)[9]) {
  if (!GEN) {
    const uint32_t *w0 = reinterpret_cast<const uint32_t *>(sgrid + base);
    const uint32_t *wp = w0 + rot;
#pragma unroll
    for (int j = 0; j < 7; j++) v[j] = wp[j];
    v[7] = wp[7 - 8 * rot];
    v[8] = W9 ? w0[8] : 0u;
  } else {
    const uint8_t *p = sgrid + base;
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = *reinterpret_cast<const uint32_t *>(p + loff[j]);
    v[8] = W9 ? *reinterpret_cast<const uint32_t *>(p + 32) : 0u;
  }
}

template <bool W9>
__device__ __forceinline__ void win_accumulate2(const uint32_t (&v1)[9], const uint32_t (&v2)[9], uint32_t (&lo)[9],
                                                uint32_t (&hi)[9]) {
#pragma unroll
  for (int q = 0; q < (W9 ? 9 : 8); q++) {
    const uint32_t w = v1[q] + v2[q];      // packed bytes, each <= 254
    lo[q] += w;                            // all four bytes, carries included: bytes 0, 2 recovered at the flush
    hi[q] += __byte_perm(w, 0u, 0x4341);   // bytes 1, 3 -> u16 lanes
  }
}

// all beams of one alignment class; count is a multiple of 4.  CHECK = per-row range test (edge beams).
template <int SH, int STRIDE, bool CHECK, bool W9, bool GEN>
__device__ __forceinline__ void win_class(const uint8_t *__restrict__ sgrid, const int32_t *__restrict__ list,
                                          int count, int lane, int hi_half, const int (&loff)[8], int bias, int row_delta,
                                          int data_size, int32_t *__restrict__ s_off, uint32_t (&lo)[9],
                                          uint32_t (&hi)[9], uint32_t (&acc)[32], int &pending) {
  for (int ib = 0; ib < count; ib += 32) {
    const int cnt = min(32, count - ib);
    __syncwarp();
    s_off[lane] = (lane < cnt) ? __ldg(list + ib + lane) : 0;  // this warp's staging row
    __syncwarp();
    if (pending + cnt > WIN_FLUSH_BEAMS) {
      win_flush<SH, STRIDE, GEN>(lo, hi, acc, hi_half);
      pending = 0;
    }
    pending += cnt;
    for (int j = 0; j < cnt; j += 4) {
      const int4 a = *reinterpret_cast<const int4 *>(s_off + j);  // one broadcast load: four window origins
      int b0, b1, b2, b3;
      if (CHECK) {
        const int32_t i0 = a.x + row_delta, i1 = a.y + row_delta, i2 = a.z + row_delta, i3 = a.w + row_delta;
        b0 = (((uint32_t)i0 + 35u) < ((uint32_t)data_size + 35u)) ? (i0 + (bias - SH)) : 0;
        b1 = (((uint32_t)i1 + 35u) < ((uint32_t)data_size + 35u)) ? (i1 + (bias - SH)) : 0;
        b2 = (((uint32_t)i2 + 35u) < ((uint32_t)data_size + 35u)) ? (i2 + (bias - SH)) : 0;
        b3 = (((uint32_t)i3 + 35u) < ((uint32_t)data_size + 35u)) ? (i3 + (bias - SH)) : 0;
      } else {
        const int lane_const = row_delta + bias - SH;
        b0 = a.x + lane_const; b1 = a.y + lane_const; b2 = a.z + lane_const; b3 = a.w + lane_const;
      }
      uint32_t v1[9], v2[9];
      win_load<W9, GEN>(sgrid, b0, hi_half, loff, v1);
      win_load<W9, GEN>(sgrid, b1, hi_half, loff, v2);
      win_accumulate2<W9>(v1, v2, lo, hi);
      win_load<W9, GEN>(sgrid, b2, hi_half, loff, v1);
      win_load<W9, GEN>(sgrid, b3, hi_half, loff, v2);
      win_accumulate2<W9>(v1, v2, lo, hi);
    }
  }
}

template <int SH, int STRIDE, bool GEN>
__device__ __forceinline__ void win_class_pair(const uint8_t *__restrict__ sgrid, const int32_t *__restrict__ li,
                                               int ci, const int32_t *__restrict__ le, int ce, int cols, int lane,
                                               int hi_half, const int (&loff)[8], int row_delta, int bias, int data_size, int32_t *__restrict__ s_off,
                                               uint32_t (&lo)[9], uint32_t (&hi)[9], uint32_t (&acc)[32]) {
  int pending = 0;
  if (SH + STRIDE * (cols - 1) + 1 > 32) {  // the last candidates need aligned word 8
    win_class<SH, STRIDE, false, true, GEN>(sgrid, li, ci, lane, hi_half, loff, bias, row_delta, data_size, s_off, lo, hi, acc, pending);
    win_class<SH, STRIDE, true, true, GEN>(sgrid, le, ce, lane, hi_half, loff, bias, row_delta, data_size, s_off, lo, hi, acc, pending);
  } else {
    win_class<SH, STRIDE, false, false, GEN>(sgrid, li, ci, lane, hi_half, loff, bias, row_delta, data_size, s_off, lo, hi, acc, pending);
    win_class<SH, STRIDE, true, false, GEN>(sgrid, le, ce, lane, hi_half, loff, bias, row_delta, data_size, s_off, lo, hi, acc, pending);
  }
  win_flush<SH, STRIDE, GEN>(lo, hi, acc, hi_half);
}

// What one k_reduce launch does: the whole tail of a CorrelateScan, or one phase of a sweep whose angles are split over
// several GPUs (b2s_matcher_correlate_split_*).  The phases are ordered: the first two compute the best response.
enum ReducePhase : int {
  REDUCE_WHOLE = 0,
  REDUCE_SPLIT_BEST = 1,    // this angle subset's best response and per-cell maxima
  REDUCE_SPLIT_TIES = 2,    // tie sums {x, y, cos, sin, count} against the global best
  REDUCE_SPLIT_FINISH = 3,  // mean pose and covariance from the global best, tie sums and maxima plane
};

struct ReduceArgs {
  const int32_t *sums;
  const double *centers;
  int32_t *flags;
  b2s_matcher_params p;
  b2s_search s;
  b2s_grid_info g;
  double scale;
  int n, nx, ny, na;
  double *probs_all;
  b2s_match_result *results;
  int k_first;
  ReducePhase phase;
  double *part_best;
  const double *glob_best;
  double *tie_out;
  const double *tie_in;
  const uint8_t *keep;  // [B][na] angles swept by a pruned sweep (nullptr: every angle); k_reduce walks only those
};


template <int STRIDE, bool GEN, bool LISTED>
__global__ void __launch_bounds__(WIN_THREADS, 1)
    k_sweep_window(const uint8_t *__restrict__ grids, size_t grid_pitch, int data_size, int copy_bytes,
                   const int32_t *__restrict__ lists, const int32_t *__restrict__ counts,
                   const int32_t *__restrict__ starts, const int32_t *__restrict__ flags, int batch, int n, int na,
                   int nx, int ny, int width_step, int32_t *__restrict__ sums, int *__restrict__ work_counter,
                   int band_rows, int nbands, int band_bytes, int neg_bands, const int32_t *__restrict__ angles,
                   const int32_t *__restrict__ n_angles, int acc_slots) {
  // LISTED (a pruned sweep: one stride-1 32 x 32 tile, nbands == 1, SweepPlan::prune): match b sweeps only the
  // n_angles[b] angles angles[b * na + ...], each split into listed_chunks beam ranges (karto_sweep_plan.cuh).  With
  // more than one range, the CTA zeroes one ny x nx plane of int32 per listed angle after the image (while its copy is
  // in flight), every item adds its rows there with shared-memory atomics (integer sums commute: the volume is the
  // same), and the planes are written out once the match's items are done.
  // Grids larger than shared memory are swept in `nbands` row bands: a work unit is (match, band, 32-row candidate
  // tile); the image holds the rows that tile of a window whose ORIGIN lies in the band can touch (band_rows +
  // STRIDE * 31 + 2), k_offsets_sorted grouped the beams by the band of their origin (bands [0, neg_bands) hold origins
  // BELOW the grid, whose upper tiles still reach it), and the partial sums of the bands are combined with RED.ADD.
  extern __shared__ __align__(128) unsigned char smem[];
  uint8_t *sgrid = smem;  // [WIN_GUARD zeros][band image][WIN_GUARD zeros]
  __shared__ uint64_t bar;
  __shared__ int s_unit, s_item;
  __shared__ __align__(16) int32_t s_offsets[WIN_THREADS / 32][32];  // per-warp staging of 32 window origins

  const int lane = threadIdx.x & 31;
  int32_t *s_off = s_offsets[threadIdx.x >> 5];
  constexpr int CPT = 32 / STRIDE;  // candidates per tile row (a tile row is always 32 bytes)
  const int tiles_x = (nx + CPT - 1) / CPT, tiles_y = (ny + 31) >> 5;
  const int unit_tiles_y = nbands > 1 ? tiles_y : 1;        // banded: one row tile per unit
  // word rotation of this lane (see win_load): lanes whose rows start in the same bank get different rotations
  int hi_half = lane >> 4;
  int loff[8];
  if (GEN) {
    const int step = ((width_step >> 2) * STRIDE) & 31;
    const int m = step ? (step & -step) : 32;  // gcd(step, 32): lanes L and L + 32/m share a row-start bank
    hi_half = ((lane * m) >> 5) & 7;
  }
#pragma unroll
  for (int j = 0; j < 8; j++) loff[j] = 4 * ((j + hi_half) & 7);
  const int list_cap = n + LIST_PAD * nbands;
  const int ngroups = 8 * nbands;

  for (int i = threadIdx.x; i < WIN_GUARD / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(sgrid)[i] = 0;  // leading guard
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint32_t parity = 0;

  while (true) {
    if (threadIdx.x == 0) {
      s_unit = atomicAdd(work_counter, 1);
      s_item = 0;
    }
    __syncthreads();
    const int unit = s_unit;
    if (unit >= batch * nbands * unit_tiles_y) break;
    const int b = unit / (nbands * unit_tiles_y), band = (unit / unit_tiles_y) % nbands, unit_ty = unit % unit_tiles_y;
    const int f = flags[b];
    const int na_b = LISTED ? n_angles[b] : na;
    if ((f & 2) || !(f & 1) || na_b == 0) {  // out-of-range lattice (error), irregular lattice (generic kernel takes it)
      __syncthreads();
      continue;
    }
    const int chunks = LISTED ? listed_chunks(na_b, n, WIN_THREADS / 32, acc_slots) : 1;
    const int items = LISTED ? na_b * chunks : na_b * tiles_x * (nbands > 1 ? 1 : tiles_y);
    int32_t *s_acc = reinterpret_cast<int32_t *>(smem + 2 * WIN_GUARD + copy_bytes);  // LISTED: [na_b][ny][nx]
    const int plane = nx * ny;
    // first / one-past-last grid row of this unit's image (the whole grid when nbands == 1)
    const int row0 = (band - neg_bands) * band_rows + STRIDE * unit_ty * 32;
    const int lo_row = max(row0, 0);
    const int band_lo = lo_row * width_step;  // flat index of the first staged byte (multiple of 16)
    int bytes = nbands > 1 ? min((((row0 - lo_row) * width_step + band_bytes) + 15) & ~15, copy_bytes - band_lo) : copy_bytes;
    if (nbands > 1) {
      // nothing to do when the image misses the grid or no beam of any angle has its origin in this band
      int any = 0;
      if (bytes > 0)
        for (int i = threadIdx.x; i < na * 8; i += blockDim.x) any |= counts[((size_t)b * na + (i >> 3)) * ngroups + band * 8 + (i & 7)];
      if (!__syncthreads_or(any)) continue;
    }
    // ---- stage this unit's band image: TMA bulk copies, 32 KB each, one mbarrier phase ----
    if (threadIdx.x == 0) {
      fence_proxy_async();  // earlier generic-proxy reads of sgrid are ordered before the async-proxy writes
      mbar_expect_tx(&bar, (uint32_t)bytes);
      const uint8_t *src = grids + (size_t)b * grid_pitch + band_lo;
      for (int off = 0; off < bytes; off += 32768) {
        int len = min(32768, bytes - off);
        bulk_g2s(sgrid + WIN_GUARD + off, src + off, (uint32_t)len, &bar);
      }
    }
    if (threadIdx.x < WIN_GUARD / 4) reinterpret_cast<uint32_t *>(sgrid + WIN_GUARD + bytes)[threadIdx.x] = 0;  // trailing guard
    if (LISTED && chunks > 1)
      for (int i = threadIdx.x; i < na_b * plane; i += blockDim.x) s_acc[i] = 0;
    mbar_wait(&bar, parity);
    parity ^= 1;
    __syncthreads();
    const int bias = WIN_GUARD - band_lo;

    int32_t *bsums = sums + (size_t)b * na * nx * ny;
    while (true) {
      int item = 0;
      if (lane == 0) item = atomicAdd(&s_item, 1);
      item = __shfl_sync(0xffffffffu, item, 0);
      if (item >= items) break;
      int k, ty, tx, j = 0, c = 0;
      if (LISTED) {
        j = item / chunks; c = item - j * chunks;
        k = angles[(size_t)b * na + j]; ty = 0; tx = 0;
      } else if (nbands > 1) {
        k = item / tiles_x; tx = item % tiles_x; ty = unit_ty;
      } else {
        k = item / (tiles_x * tiles_y);
        const int t = item % (tiles_x * tiles_y);
        ty = t / tiles_x; tx = t % tiles_x;
      }
      const int row_delta = STRIDE * (ty * 32 + lane) * width_step + tx * 32;  // this lane's row start relative to a beam's origin
      const int32_t *list = lists + ((size_t)b * na + k) * list_cap;
      const int32_t *cn = counts + ((size_t)b * na + k) * ngroups + band * 8;
      const int32_t *sg = starts + ((size_t)b * na + k) * ngroups + band * 8;

      uint32_t acc[32];
#pragma unroll
      for (int j = 0; j < 32; j++) acc[j] = 0;
      uint32_t lo[9], hi[9];
#pragma unroll
      for (int j = 0; j < 9; j++) { lo[j] = 0; hi[j] = 0; }
      // groups of this band: I0 I1 I2 I3 E0 E1 E2 E3 (interior / edge beams of each alignment class)
      const int cols = min(CPT, nx - tx * CPT);
      if (LISTED) {  // this item's range of the concatenated groups
        int r0, r1, off[8], len[8];
        chunk_range(cn[0] + cn[1] + cn[2] + cn[3] + cn[4] + cn[5] + cn[6] + cn[7], c, chunks, r0, r1);
        chunk_groups(cn, r0, r1, off, len);
        win_class_pair<0, STRIDE, GEN>(sgrid, list + sg[0] + off[0], len[0], list + sg[4] + off[4], len[4], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<1, STRIDE, GEN>(sgrid, list + sg[1] + off[1], len[1], list + sg[5] + off[5], len[5], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<2, STRIDE, GEN>(sgrid, list + sg[2] + off[2], len[2], list + sg[6] + off[6], len[6], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<3, STRIDE, GEN>(sgrid, list + sg[3] + off[3], len[3], list + sg[7] + off[7], len[7], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
      } else {
        win_class_pair<0, STRIDE, GEN>(sgrid, list + sg[0], cn[0], list + sg[4], cn[4], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<1, STRIDE, GEN>(sgrid, list + sg[1], cn[1], list + sg[5], cn[5], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<2, STRIDE, GEN>(sgrid, list + sg[2], cn[2], list + sg[6], cn[6], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
        win_class_pair<3, STRIDE, GEN>(sgrid, list + sg[3], cn[3], list + sg[7], cn[7], cols, lane, hi_half, loff, row_delta, bias, data_size, s_off, lo, hi, acc);
      }

      // ---- write / accumulate this lane's row ----
      const int iy = ty * 32 + lane;
      if (iy < ny) {
        int32_t *dst = bsums + ((size_t)k * ny + iy) * nx + tx * CPT;
        if (LISTED && chunks > 1) {
          int32_t *sdst = s_acc + (j * ny + iy) * nx;  // lane r's row: banks (r * nx + x) mod 32
#pragma unroll
          for (int x = 0; x < CPT; x++)
            if (x < nx && acc[x]) atomicAdd(sdst + x, (int32_t)acc[x]);
        } else if (nbands == 1) {
#pragma unroll
          for (int x = 0; x < CPT; x++)
            if (tx * CPT + x < nx) dst[x] = (int32_t)acc[x];
        } else {
#pragma unroll
          for (int x = 0; x < CPT; x++)
            if (tx * CPT + x < nx && acc[x]) atomicAdd(dst + x, (int32_t)acc[x]);
        }
      }
    }
    __syncthreads();  // everyone is done with sgrid before the next unit's copy is issued
    if (LISTED && chunks > 1)  // (the next unit zeroes the planes only after its own __syncthreads)
      for (int i = threadIdx.x; i < na_b * plane; i += blockDim.x) {
        const int jj = i / plane;
        bsums[(size_t)angles[(size_t)b * na + jj] * plane + (i - jj * plane)] = s_acc[i];
      }
  }
}

// ----------------------------------------------------------------------------------------------
// k_reduce: the fp64 tail of CorrelateScan (Mapper.cpp:397-523): penalties, best response, per-cell maxima,
// tie-averaged pose, positional covariance.  One CTA per match.  Candidate order of the reference is
// (iy, ix, k) with linear index (iy*nx + ix)*na + k; ties are summed sequentially in that order when there are
// at most RED_MAX_TIES of them (bit-identical to the reference), otherwise by a fixed-order tree.
// ----------------------------------------------------------------------------------------------
constexpr int RED_THREADS = 512;
// (two CTAs per SM, so one match's serial tail overlaps another's streaming pass)
constexpr int RED_MAX_TIES = 512;
constexpr int RED_UNROLL = 8;

__device__ __forceinline__ double candidate_response(int32_t isum, int n, bool do_penalize, double sq_xy,
                                                     double angle, double center_h, const b2s_matcher_params &p) {
  double response = (double)isum;
  response /= (double)((uint32_t)n * (uint32_t)GRID_OCCUPIED);  // Mapper.cpp:852
  if (do_penalize && !double_equal(response, 0.0)) {
    double dpen = 1.0 - (DISTANCE_PENALTY_GAIN * sq_xy / p.distance_variance_penalty);
    dpen = dmax(dpen, p.minimum_distance_penalty);
    double sq_a = (angle - center_h) * (angle - center_h);
    double apen = 1.0 - (ANGLE_PENALTY_GAIN * sq_a / p.angle_variance_penalty);
    apen = dmax(apen, p.minimum_angle_penalty);
    response *= (dpen * apen);
  }
  return response;
}

// The float pre-filter of k_reduce and k_prune_select.  apf[k] = anglePenalty(k) / (N * 100) for the angles
// [0, na) of the launch (k_first + k of the search), the cell factor is red_dist_factor, and red_fscore is a candidate's
// float score: relative error < 3e-7 vs candidate_response.  A candidate whose score is below red_margin(largest
// score) cannot have the largest exact response; ambiguous ones (unpenalised response near the 1e-6 DoubleEqual
// threshold of the penalty test, Mapper.cpp:399) must always be evaluated exactly.
__device__ __forceinline__ void red_angle_factors(float *apf, int na, int k_first, double start_a, double center_h,
                                                  double D, bool do_penalize, const b2s_search &s,
                                                  const b2s_matcher_params &p) {
  for (int k = threadIdx.x; k < na; k += blockDim.x) {
    double apen = 1.0;
    if (do_penalize) {
      const double angle = start_a + (double)(uint32_t)(k_first + k) * s.angle_res;
      apen = dmax(1.0 - (ANGLE_PENALTY_GAIN * ((angle - center_h) * (angle - center_h)) / p.angle_variance_penalty), p.minimum_angle_penalty);
    }
    apf[k] = (float)(apen / D);
  }
}

__device__ __forceinline__ float red_dist_factor(double sq_xy, const b2s_matcher_params &p) {
  return (float)dmax(1.0 - (DISTANCE_PENALTY_GAIN * sq_xy / p.distance_variance_penalty), p.minimum_distance_penalty);
}

__device__ __forceinline__ float red_fscore(int32_t isum, float apf_k, float dpf, float inv_d, bool do_penalize,
                                            bool &ambiguous) {
  const float u = (float)isum * inv_d;  // unpenalised response
  ambiguous = (u > 0.5e-6f) && (u < 2.0e-6f);
  if (!do_penalize || u <= 1.0e-6f) return u;
  return (float)isum * apf_k * dpf;
}

__device__ __forceinline__ float red_margin(float fmax) { return fmax * (1.0f - 2.0e-6f) - 1.0e-30f; }

// ----------------------------------------------------------------------------------------------
// Angle pruning (SweepPlan::prune: one 32 x 32 stride-1 tile, the whole grid in shared memory, a whole search).
//
// CorrelateScan needs exact responses only for the best candidate, its DoubleEqual ties (1e-6) and the per-cell
// maxima that reach best - 0.1 (the only cells ComputePositionalCovariance reads, Mapper.cpp:586).  A candidate whose
// response is below best - 0.1 is none of these, and leaving it out cannot lower a cell maximum that reaches best - 0.1.
// So an angle may be skipped when an upper bound of all its responses is below L - 0.1 for some lower bound L <= best:
//   k_sweep_bound   UBr(k) = max over 8 x 8 blocks of 4 x 4 candidates of
//                   (SUM_beams P[a_i + block corner]) / (N * 100) * (max distance penalty of the block * anglePenalty(k)),
//                   P the 4x4 max-pooled grid (k_grid_pool), summed over the beams the exact sweep's lists hold, placed
//                   by the bound itself (beams dropped as empty windows add 0 everywhere).  Same fp64 operations as
//                   candidate_response, so UBr(k) >= every response of angle k.  No window lists exist yet:
//                   k_offsets_sorted lists only the angles of the two exact passes below.
//                   UBr is computed only where it can matter: a group pass bounds BOUND_GROUP consecutive angles at
//                   once from a 7x7 pooled image, and the rounds below bound single angles only in groups whose bound
//                   reaches what they are compared with (see k_sweep_bound's modes).
//   probe           the PRUNE_PROBE angles with the largest UBr are swept exactly (k_sweep_window on an angle list);
//   k_prune_select  L = the largest exact response among them (a real candidate, so L <= best; only the candidates
//                   k_reduce's float pre-filter leaves are evaluated exactly); every other angle is
//                   swept iff UBr(k) >= L - 0.1 - 1e-9.  When L - 0.1 is near 0 (within the 1e-6 band in which a
//                   response is not penalised, Mapper.cpp:399) every angle is swept.
// k_reduce walks only the swept angles (the others would read 0); the response volume is completed on request
// (get_response_sums).
// ----------------------------------------------------------------------------------------------
// bytes c .. c + 3 of the 8 bytes hi:lo, c = sel % 4 (prmt's forward-4-extract mode reads only sel's two low bits)
__device__ __forceinline__ uint32_t extract4(uint32_t lo, uint32_t hi, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32.f4e %0, %1, %2, %3;" : "=r"(d) : "r"(lo), "r"(hi), "r"(sel));
  return d;
}

// the 8 pooled bytes of block row `rw / width_step` of an interior beam whose block (0, 0) corner is at byte `addr` of
// the staged image: P at block columns 0..3 (lo) and 4..7 (hi) in byte order.  rw % 8 == 0, so every row of the beam
// has the alignment of addr.
__device__ __forceinline__ void bound_row(const uint8_t *__restrict__ pb, int addr, int rw, uint32_t &lo,
                                          uint32_t &hi) {
  const uint32_t *w = reinterpret_cast<const uint32_t *>(pb + ((addr + rw) & ~3));
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
  lo = extract4(w0, w1, (uint32_t)addr);
  hi = extract4(w1, w2, (uint32_t)addr);
}

constexpr int BOUND_FLUSH = 64 * 32;  // beams placed between flushes of k_sweep_bound's packed corner sums

// What one launch of k_sweep_bound computes (see the angle-pruning comment above):
//   BOUND_GROUPS  gub[b][g] = a bound of UBr over the BOUND_GROUP consecutive angles of group g, from the 7x7 image P7
//   BOUND_PROBE   UBr for the top groups by gub (at least PRUNE_PROBE angles), f16 = the PRUNE_PROBE-th largest of
//                 them, UBr for every other group whose gub reaches f16, then the probe list: the PRUNE_PROBE largest
//                 UBr of all evaluated angles (ties: lower index).  Every angle not evaluated has UBr <= gub < f16,
//                 so this is the top PRUNE_PROBE of every angle's UBr.
//   BOUND_SELECT  UBr for the angles k_prune_select listed (groups not yet evaluated whose gub reaches the cut), and
//                 of those, the ones whose UBr reaches the cut join the kept list
enum { BOUND_GROUPS = 0, BOUND_PROBE = 1, BOUND_SELECT = 2 };

// One persistent CTA per match at a time (like k_sweep_window): the pooled image (its four residue planes, see
// pool_index) is staged by TMA, warps take items of units (an angle, or a group of BOUND_GROUP angles).  A round of
// few units cuts each unit's beams into ranges (bound_chunks / bound_range in karto_sweep_plan.cuh), and each item
// adds its 64 block sums into the unit's u32 row in shared memory; after a __syncthreads one warp per unit scores the
// row.  Integer sums commute, so the value is the one a single pass over the beams gives.  The bound reads no window
// lists: for each item a warp places 32 beams at a time, one per lane, and compacts the interior and the edge ones
// into its staging row.
//   One angle: the beam's window origin and class by win_origin_class (the definition k_offsets_sorted lists them
//   by), dropping the ones the lists would drop.  Which beams add is the same set as in the lists and integer sums
//   commute, so UBr is the one the lists would give.
//   A group: the beam's origins at the group's angles are bracketed per axis in fp32 with a margin far above fp32's
//   error (a beam's lookup value is a few hundred cells at most), rounded outwards the way kround can round.  When
//   both brackets span at most BOUND_SPREAD cells, the beam adds P7 at the bracket's low corner: P7 there covers P at
//   every member's origin, flat index and row wrap included.  Otherwise (long ranges, coarse angle steps, far or
//   non-finite points) the beam adds the largest P7 over the members' exact origins.  Beams whose windows are empty
//   are kept (they only loosen the bound), and the range test decides edge beams as before.
//
// Interior beams, four at a time: lane L = slot * 8 + row takes beam `slot` of the four and adds its 8 block corners
// of block row `row` (8 contiguous plane bytes) as two words, one byte per block column.  Two beams' words add
// bytewise without carry (the window kernel runs only on grids of bytes <= 127, so P, P7 <= 127), and each pair goes
// into a plain u32 sum and, through one byte permute, a sum of bytes 1 and 3 in u16 lanes; the plain sum less the
// latter shifted by 8 leaves bytes 0 and 2 in u16 lanes.  A slot takes at most 8 beams per 32 placed, 8 x 127 per u16
// lane, so the sums are flushed into the per-column u32 totals every BOUND_FLUSH beams placed (64 x 1016 < 65536)
// and at the end of the item's range.  The totals of the four slots are then summed by shuffles so that lane L ends with
// blocks (L % 8, 2 (L / 8)) and (L % 8, 2 (L / 8) + 1).  Edge beams and the last 0..3 interior ones read P byte by
// byte with the range test, at the lane's own two blocks (the value of an interior one is the same either way).
// The value of a unit is candidate_response's fp64 operations on the block's sum, the block's largest distance
// penalty and the unit's largest angle penalty, so it is at least every response of every angle of the unit.
// STAGE (SweepPlan::bound_stage / group_stage): the scan-local points (and for single angles the summed-area table)
// sit in shared memory after the pooled image; otherwise they are read from global memory through L1.  The `rows`
// unit rows follow (SweepPlan::bound_rows / group_rows).
template <bool STAGE, int MODE>
__global__ void __launch_bounds__(WIN_THREADS, 1)
    k_sweep_bound(const uint8_t *__restrict__ pools, size_t pool_pitch_, int pool_bytes_, int plane, int lead,
                  const double *__restrict__ local, const double *__restrict__ grid_off,
                  const int32_t *__restrict__ bases, const uint16_t *__restrict__ sat_all, int sbx, int sby,
                  int height, int rows_total, int cols_total, double scale, const int32_t *__restrict__ flags,
                  const double *__restrict__ centers, b2s_matcher_params p, b2s_search s, int batch, int n, int na,
                  int nx, int ny, int width_step, int data_size, double *__restrict__ ubr, double *__restrict__ gub,
                  int32_t *__restrict__ angles, int32_t *__restrict__ n_angles, uint8_t *__restrict__ keep,
                  const int32_t *__restrict__ n_eval, const double *__restrict__ cuts,
                  unsigned long long *__restrict__ pruned_total, int32_t *__restrict__ scratch, int rows,
                  int *__restrict__ work_counter) {
  constexpr bool GRP = MODE == BOUND_GROUPS;
  constexpr int NJ = GRP ? BOUND_GROUP : 1;  // angles per unit
  // [WIN_GUARD zeros][pooled image][WIN_GUARD zeros] (+ STAGE: [n] x, [n] y of the scan-local points, the SAT)
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t bar;
  __shared__ int s_unit, s_cnt, s_top;
  __shared__ double s_f16;
  __shared__ __align__(16) int32_t s_offsets[WIN_THREADS / 32][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int32_t *s_off = s_offsets[warp];
  const bool pen = s.do_penalize != 0;
  const int SW = sbx + 1;
  const int sat_len = ((sby + 1) * SW + 7) & ~7;  // entries per match, padded to 16 bytes
  const int ng = (na + BOUND_GROUP - 1) / BOUND_GROUP;
  // the match's list of angles to bound and (BOUND_PROBE) its groups by bound, largest first, in global memory
  // (scratch[b][na + ng]): shared memory beside the pooled image is budgeted for k_sweep_window's static arrays only
  double *s_lx = reinterpret_cast<double *>(smem + WIN_GUARD + pool_bytes_ + WIN_GUARD), *s_ly = s_lx + n;
  uint16_t *s_sat = reinterpret_cast<uint16_t *>(s_ly + n);
  uint32_t *s_rows = STAGE ? reinterpret_cast<uint32_t *>(s_sat + (sat_all ? sat_len : 0)) : reinterpret_cast<uint32_t *>(s_lx);
  const unsigned lanes_below = (1u << lane) - 1u;
  // the largest distance penalty of the candidates of block (by, bx), as k_reduce computes sq and candidate_response
  // the penalty (-1: the block holds no candidate)
  auto block_dpen = [&](int by, int bx) {
    double mx = -1.0;
    for (int iy = 4 * by; iy < min(4 * by + 4, ny); iy++)
      for (int ix = 4 * bx; ix < min(4 * bx + 4, nx); ix++) {
        const double y = -s.offset_y + (double)(uint32_t)iy * s.res_y, x = -s.offset_x + (double)(uint32_t)ix * s.res_x;
        const double sq = x * x + y * y;
        mx = dmax(mx, pen ? dmax(1.0 - (DISTANCE_PENALTY_GAIN * sq / p.distance_variance_penalty), p.minimum_distance_penalty) : 1.0);
      }
    return mx;
  };
  const int slot = lane >> 3, row = lane & 7;
  const double dpen_a = block_dpen(row, 2 * slot), dpen_b = block_dpen(row, 2 * slot + 1);
  for (int i = threadIdx.x; i < WIN_GUARD / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(smem)[i] = 0;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int off_a = 4 * row * width_step + 8 * slot, off_b = off_a + 4;  // the lane's two block corners
  const int rw = row * width_step;  // its block row in a plane
  const double D = (double)((uint32_t)n * (uint32_t)GRID_OCCUPIED);
  const uint8_t *pb = smem + WIN_GUARD;  // the staged pooled image
  const uint32_t limit = (uint32_t)(lead + data_size);
  const float scf = (float)scale;
  // P (P7) at flat index a + corner, modulo 2^32 like the reference's base + offset; 0 outside the grid
  auto pool_at = [&](int32_t a, int off) -> uint32_t {
    const uint32_t fa = (uint32_t)a + (uint32_t)off;
    return (fa + (uint32_t)lead < limit) ? pb[pool_index((int32_t)fa, lead, plane)] : 0u;
  };
  uint32_t parity = 0;
  while (true) {
    if (threadIdx.x == 0) s_unit = atomicAdd(work_counter, 1);
    __syncthreads();
    const int b = s_unit;
    if (b >= batch) break;
    const int f = flags[b];
    if ((f & 2) || !(f & 1)) {  // not swept by the window kernel: no list, every angle kept (the generic kernel)
      if (MODE == BOUND_PROBE) {
        for (int k = threadIdx.x; k < na; k += blockDim.x) keep[(size_t)b * na + k] = 1;
        if (threadIdx.x == 0) n_angles[b] = 0;
      }
      __syncthreads();
      continue;
    }
    const int nev = MODE == BOUND_SELECT ? n_eval[b] : 0;
    int32_t *s_list = scratch + (size_t)b * (na + ng), *s_order = s_list + na;
    const double *s_gub = gub + (size_t)b * ng;
    if (MODE == BOUND_SELECT && nev == 0) {  // nothing to bound: the kept list is final
      __syncthreads();
      continue;
    }
    if (threadIdx.x == 0) {
      fence_proxy_async();
      mbar_expect_tx(&bar, (uint32_t)pool_bytes_);
      const uint8_t *src = pools + (size_t)b * pool_pitch_;
      for (int off = 0; off < pool_bytes_; off += 32768)
        bulk_g2s(smem + WIN_GUARD + off, src + off, (uint32_t)min(32768, pool_bytes_ - off), &bar);
    }
    if (threadIdx.x < WIN_GUARD / 4) reinterpret_cast<uint32_t *>(smem + WIN_GUARD + pool_bytes_)[threadIdx.x] = 0;
    const double *g_pts = local + (size_t)b * n * 2;
    const uint16_t *g_sat = sat_all ? sat_all + (size_t)b * sat_len : nullptr;
    if (STAGE) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        s_lx[i] = g_pts[2 * i];
        s_ly[i] = g_pts[2 * i + 1];
      }
      if (sat_all)
        for (int i = threadIdx.x; i < sat_len / 8; i += blockDim.x)
          reinterpret_cast<uint4 *>(s_sat)[i] = reinterpret_cast<const uint4 *>(g_sat)[i];
    }
    if (MODE == BOUND_PROBE) {  // round (a): the top groups by bound, until they hold PRUNE_PROBE angles
      for (int k = threadIdx.x; k < na; k += blockDim.x) ubr[(size_t)b * na + k] = __longlong_as_double(0x7ff8000000000000ll);
      __syncthreads();
      for (int g = threadIdx.x; g < ng; g += blockDim.x) {
        const double u = s_gub[g];
        int rank = 0;
        for (int h = 0; h < ng; h++) rank += (s_gub[h] > u) || (s_gub[h] == u && h < g);
        s_order[rank] = g;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int cnt = 0, r = 0;
        while (cnt < min(PRUNE_PROBE, na)) {
          const int g = s_order[r++];
          for (int k = g * BOUND_GROUP; k < min(g * BOUND_GROUP + BOUND_GROUP, na); k++) s_list[cnt++] = k;
        }
        s_top = r;
        s_cnt = cnt;
      }
    } else if (MODE == BOUND_SELECT) {  // the list k_prune_select left at the end of the match's angle list
      for (int j = threadIdx.x; j < nev; j += blockDim.x) s_list[j] = angles[(size_t)b * na + na - nev + j];
    }
    const WinGeom G = win_geom(grid_off[2 * b], grid_off[2 * b + 1], scale, bases[(size_t)b * nx * ny], 1, rows_total,
                               cols_total, width_step, data_size, height, nx, ny, 1, 1, 0);
    // fp32 margin of a group's origin brackets, in cells: fp32's error of the rotation and of the products (far below
    // 1e-5 of |x| + |y| in cells) and the (o + gridOffset) - gridOffset double rounding of the exact lookup value
    const float mg_match = 4e-3f + (float)(1e-15 * (fabs(G.gox) + fabs(G.goy)) * scale);
    mbar_wait(&bar, parity);
    parity ^= 1;
    __syncthreads();
    const double ch = centers[3 * b + 2];

    // the largest angle penalty of angles k0 .. k0 + cnt - 1 (cnt = 1 unless GRP)
    auto unit_apen = [&](int k0, int cnt) -> double {
      double apen = GRP ? -1.0 : 1.0;
      if (pen)
#pragma unroll
        for (int j = 0; j < NJ; j++) {
          const double angle = win_angle(ch, s.angle_offset, s.angle_res, k0 + min(j, cnt - 1));
          const double sq_a = (angle - ch) * (angle - ch);
          const double ap = dmax(1.0 - (ANGLE_PENALTY_GAIN * sq_a / p.angle_variance_penalty), p.minimum_angle_penalty);
          apen = GRP ? dmax(apen, ap) : ap;
        }
      return apen;
    };
    // candidate_response's operations, with the block's largest sum and largest distance penalty: the bound of a unit
    // whose block sums are ua, ub in every lane (see bound_sums), in every lane
    auto bound_value = [&](uint32_t ua, uint32_t ub, double apen) -> double {
      double r = -1.0;
      if (dpen_a >= 0.0) r = dmax(r, pen ? ((double)ua / D) * (dpen_a * apen) : (double)ua / D);
      if (dpen_b >= 0.0) r = dmax(r, pen ? ((double)ub / D) * (dpen_b * apen) : (double)ub / D);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) r = dmax(r, __shfl_xor_sync(0xffffffffu, r, d));
      return r;
    };
    // the sums of beams [i_lo, i_hi) (i_lo % 32 == 0) of angles k0 .. k0 + cnt - 1 at the lane's blocks
    // (L % 8, 2 (L / 8)) -> ua and (L % 8, 2 (L / 8) + 1) -> ub
    auto bound_sums = [&](int k0, int cnt, int i_lo, int i_hi, uint32_t &ua, uint32_t &ub) {
      double cd[NJ], sd[NJ];
      float cf[NJ], sf[NJ];
#pragma unroll
      for (int j = 0; j < NJ; j++) {
        const double angle = win_angle(ch, s.angle_offset, s.angle_res, k0 + min(j, cnt - 1));
        cd[j] = cos(angle);
        sd[j] = sin(angle);
        cf[j] = (float)cd[j];
        sf[j] = (float)sd[j];
      }
      ua = 0;                                   // the lane's two blocks, beams read with the range test
      ub = 0;
      uint32_t s0 = 0, s1 = 0, o0 = 0, o1 = 0;  // interior pairs: plain sums and byte 1 / 3 sums of columns 0..3, 4..7
      uint32_t t[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // interior totals of the lane's slot and row, per block column
      for (int i0 = i_lo; i0 < i_hi; i0 += 32) {
        const int i = i0 + lane;
        int cls = 255;
        int32_t a = 0;
        bool fb = false;           // GRP: the beam adds the largest P7 over its members' exact origins ...
        int32_t fa[NJ];            // ... these (WIN_SKIP: the member's window is wholly outside the grid)
        if (i < i_hi) {
          const double plx = STAGE ? s_lx[i] : __ldg(g_pts + 2 * i), ply = STAGE ? s_ly[i] : __ldg(g_pts + 2 * i + 1);
          if (!GRP) {
            bool empty;
            cls = win_origin_class(plx, ply, cd[0], sd[0], G, sat_all != nullptr, STAGE ? s_sat : g_sat, SW, a, empty);
          } else {
            const float px = (float)plx, py = (float)ply;
            float xl = INFINITY, xh = -INFINITY, yl = INFINITY, yh = -INFINITY;
#pragma unroll
            for (int j = 0; j < NJ; j++) {
              const float x = cf[j] * px - sf[j] * py, y = sf[j] * px + cf[j] * py;
              xl = fminf(xl, x); xh = fmaxf(xh, x); yl = fminf(yl, y); yh = fmaxf(yh, y);
            }
            const float mg = mg_match + 1e-5f * (fabsf(px) + fabsf(py)) * scf;
            xl = xl * scf - mg; xh = xh * scf + mg; yl = yl * scf - mg; yh = yh * scf + mg;
            // kround(v) lies in [ceil(v - 0.5), floor(v + 0.5)], both monotone in v
            if (fabsf(xl) < 8192.f && fabsf(xh) < 8192.f && fabsf(yl) < 8192.f && fabsf(yh) < 8192.f) {
              const int mx = (int)ceilf(xl - 0.5f), Mx = (int)floorf(xh + 0.5f);
              const int my = (int)ceilf(yl - 0.5f), My = (int)floorf(yh + 0.5f);
              if (Mx - mx <= BOUND_SPREAD && My - my <= BOUND_SPREAD) {
                a = (int32_t)((uint32_t)G.base00 + (uint32_t)mx + (uint32_t)my * (uint32_t)width_step);
                const long long last = (long long)a + 28ll * width_step + 28;  // the last corner
                if (last < -lead || a >= data_size) cls = 255;                  // every corner reads 0
                else if (a >= -lead && last <= (long long)data_size + 4 * (POOL_PAD - 8)) cls = 0;  // in the planes
                else cls = 4;
              } else {
                fb = true;
              }
            } else {
              fb = true;
            }
            if (fb) {
#pragma unroll
              for (int j = 0; j < NJ; j++) {
                int32_t aj;
                bool empty;
                const int c = j < cnt ? win_origin_class(plx, ply, cd[j], sd[j], G, false, nullptr, SW, aj, empty) : 255;
                fa[j] = c < 255 ? aj : WIN_SKIP;
              }
            }
          }
        }
        // Interior windows lie within WIN_GUARD - 16 bytes of the grid (a group's low corner: within the planes), so
        // every corner they read is inside the staged planes or their zero padding.  The staging row holds the first
        // n4 of them (a multiple of 4) as image addresses: beam q < n8 at 8 (q / 8) + 2 (q % 4) + (q / 4) % 2, so that
        // one load gives a lane its slot's two beams of a group of 8, and a last group of 4 at q.  From n4 on it holds
        // the origins of the other 0..3 and of the edge ones, padded to a multiple of 4 with an origin far outside.
        const unsigned m_int = __ballot_sync(0xffffffffu, cls < 4), m_edge = __ballot_sync(0xffffffffu, cls >= 4 && cls < 8);
        const int n_int = __popc(m_int), n8 = n_int & ~7, n4 = n_int & ~3, n_chk = n_int + __popc(m_edge) - n4;
        __syncwarp();
        if (cls < 4) {
          const int q = __popc(m_int & lanes_below);
          s_off[q < n8 ? (q & ~7) + 2 * (q & 3) + ((q >> 2) & 1) : q] = q < n4 ? pool_index(a, lead, plane) : a;
        } else if (cls < 8) {
          s_off[n_int + __popc(m_edge & lanes_below)] = a;
        }
        const int n_end = n4 + ((n_chk + 3) & ~3);
        if (lane >= n4 + n_chk && lane < n_end) s_off[lane] = WIN_SKIP;  // slots no beam was compacted into
        __syncwarp();
        for (int g = 0; g < (n8 >> 3); g++) {
          const int2 e = *reinterpret_cast<const int2 *>(s_off + 8 * g + 2 * slot);
          uint32_t xl, xh, yl, yh;
          bound_row(pb, e.x, rw, xl, xh);
          bound_row(pb, e.y, rw, yl, yh);
          xl += yl;
          xh += yh;
          s0 += xl;
          o0 += __byte_perm(xl, 0, 0x4341);
          s1 += xh;
          o1 += __byte_perm(xh, 0, 0x4341);
        }
        if (n4 & 4) {
          uint32_t xl, xh;
          bound_row(pb, s_off[n8 + slot], rw, xl, xh);
          s0 += xl;
          o0 += __byte_perm(xl, 0, 0x4341);
          s1 += xh;
          o1 += __byte_perm(xh, 0, 0x4341);
        }
        if (((i0 + 32) & (BOUND_FLUSH - 1)) == 0 || i0 + 32 >= i_hi) {
          const uint32_t e0 = s0 - (o0 << 8), e1 = s1 - (o1 << 8);  // bytes 0 and 2 in u16 lanes
          t[0] += e0 & 0xffffu; t[1] += o0 & 0xffffu; t[2] += e0 >> 16; t[3] += o0 >> 16;
          t[4] += e1 & 0xffffu; t[5] += o1 & 0xffffu; t[6] += e1 >> 16; t[7] += o1 >> 16;
          s0 = s1 = o0 = o1 = 0;
        }
        for (int j = n4; j < n_end; j += 4) {
          const int4 a4 = *reinterpret_cast<const int4 *>(s_off + j);  // one broadcast load: four window origins
          const int32_t as[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
          for (int q = 0; q < 4; q++) {
            ua += pool_at(as[q], off_a);
            ub += pool_at(as[q], off_b);
          }
        }
        if (GRP) {
          for (unsigned m_fb = __ballot_sync(0xffffffffu, fb); m_fb; m_fb &= m_fb - 1) {
            const int src = __ffs(m_fb) - 1;
            uint32_t va = 0, vb = 0;
#pragma unroll
            for (int j = 0; j < NJ; j++) {
              const int32_t aj = __shfl_sync(0xffffffffu, fa[j], src);
              va = max(va, pool_at(aj, off_a));
              vb = max(vb, pool_at(aj, off_b));
            }
            ua += va;
            ub += vb;
          }
        }
      }
      // the four slots' totals summed: lane L keeps block columns 2 (L / 8) and 2 (L / 8) + 1 of row L % 8
      {
        const bool hi16 = lane & 16, hi8 = lane & 8;
        uint32_t k4[4];
#pragma unroll
        for (int c = 0; c < 4; c++)
          k4[c] = (hi16 ? t[c + 4] : t[c]) + __shfl_xor_sync(0xffffffffu, hi16 ? t[c] : t[c + 4], 16);
#pragma unroll
        for (int c = 0; c < 2; c++) {
          const uint32_t v = (hi8 ? k4[c + 2] : k4[c]) + __shfl_xor_sync(0xffffffffu, hi8 ? k4[c] : k4[c + 2], 8);
          if (c == 0) ua += v; else ub += v;
        }
      }
    };
    // one round: the bounds of `units` units, unit u being angles k0 .. k0 + cnt - 1 (unit_of(u, k0, cnt)), handed to
    // put(u, bound) in lane 0 of one warp.  Split into ranges, the round ends with a __syncthreads.
    auto bound_round = [&](int units, auto unit_of, auto put) {
      constexpr int W = WIN_THREADS / 32;
      const int C = bound_chunks(units, n, W, rows);
      int k0, cnt;
      uint32_t ua, ub;
      if (C == 1) {
        for (int u = warp; u < units; u += W) {
          unit_of(u, k0, cnt);
          bound_sums(k0, cnt, 0, n, ua, ub);
          const double r = bound_value(ua, ub, unit_apen(k0, cnt));
          if (lane == 0) put(u, r);
        }
        return;
      }
      for (int i = threadIdx.x; i < units * 64; i += blockDim.x) s_rows[i] = 0;
      __syncthreads();
      for (int it = warp; it < units * C; it += W) {
        const int u = it / C;
        int lo, hi;
        bound_range(n, it - u * C, C, lo, hi);
        unit_of(u, k0, cnt);
        bound_sums(k0, cnt, lo, hi, ua, ub);
        atomicAdd(s_rows + 64 * u + 2 * lane, ua);
        atomicAdd(s_rows + 64 * u + 2 * lane + 1, ub);
      }
      __syncthreads();
      for (int u = warp; u < units; u += W) {
        unit_of(u, k0, cnt);
        const double r = bound_value(s_rows[64 * u + 2 * lane], s_rows[64 * u + 2 * lane + 1], unit_apen(k0, cnt));
        if (lane == 0) put(u, r);
      }
    };
    // the angles at list positions [j0, j1)
    auto bound_list = [&](int j0, int j1) {
      bound_round(
          j1 - j0, [&](int u, int &k0, int &cnt) { k0 = s_list[j0 + u]; cnt = 1; },
          [&](int u, double r) { ubr[(size_t)b * na + s_list[j0 + u]] = r; });
    };

    if (GRP) {
      bound_round(
          ng, [&](int g, int &k0, int &cnt) { k0 = g * BOUND_GROUP; cnt = min(BOUND_GROUP, na - g * BOUND_GROUP); },
          [&](int g, double r) { gub[(size_t)b * ng + g] = r; });
    } else if (MODE == BOUND_PROBE) {
      const int T = min(PRUNE_PROBE, na);
      const int n_a = s_cnt;
      bound_list(0, n_a);
      __syncthreads();
      // f16: the T-th largest bound of round (a)
      for (int j = threadIdx.x; j < n_a; j += blockDim.x) {
        const double u = ubr[(size_t)b * na + s_list[j]];
        int rank = 0;
        for (int h = 0; h < n_a; h++) {
          const double v = ubr[(size_t)b * na + s_list[h]];
          rank += (v > u) || (v == u && h < j);
        }
        if (rank == T - 1) s_f16 = u;
      }
      __syncthreads();
      // round (b): every other group whose bound reaches f16
      const double f16 = s_f16;
      for (int r = s_top + threadIdx.x; r < ng; r += blockDim.x) {
        const int g = s_order[r];
        if (s_gub[g] >= f16) {
          const int k1 = min(g * BOUND_GROUP + BOUND_GROUP, na);
          const int pos = atomicAdd(&s_cnt, k1 - g * BOUND_GROUP);
          for (int k = g * BOUND_GROUP; k < k1; k++) s_list[pos + k - g * BOUND_GROUP] = k;
        }
      }
      __syncthreads();
      const int n_ab = s_cnt;
      bound_list(n_a, n_ab);
      for (int k = threadIdx.x; k < na; k += blockDim.x) keep[(size_t)b * na + k] = 0;
      __syncthreads();
      // the probe: the T largest bounds of all evaluated angles, ties to the lower index
      for (int j = threadIdx.x; j < n_ab; j += blockDim.x) {
        const int k = s_list[j];
        const double u = ubr[(size_t)b * na + k];
        int rank = 0;
        for (int h = 0; h < n_ab; h++) {
          const int kh = s_list[h];
          const double v = ubr[(size_t)b * na + kh];
          rank += (v > u) || (v == u && kh < k);
        }
        if (rank < T) {
          angles[(size_t)b * na + rank] = k;
          keep[(size_t)b * na + k] = 1;
        }
      }
      if (threadIdx.x == 0) n_angles[b] = T;
    } else {  // BOUND_SELECT
      bound_list(0, nev);
      if (threadIdx.x == 0) s_cnt = n_angles[b];
      __syncthreads();
      const double cut = cuts[b];
      int pruned = 0;
      for (int j = threadIdx.x; j < nev; j += blockDim.x) {
        const int k = s_list[j];
        if (ubr[(size_t)b * na + k] >= cut) {
          angles[(size_t)b * na + atomicAdd(&s_cnt, 1)] = k;
          keep[(size_t)b * na + k] = 1;
        } else {
          pruned++;
        }
      }
      if (pruned) atomicAdd(pruned_total, (unsigned long long)pruned);
      __syncthreads();
      if (threadIdx.x == 0) n_angles[b] = s_cnt;
    }
    __syncthreads();  // everyone is done with the image before the next match's copy is issued
  }
}

// L from the probe's exact sums, then match b's second angle list: the angles not probed whose bound reaches
// L - 0.1 - 1e-9.  An angle the probe round did not bound (ubr NaN) has UBr <= the bound of its group: when that is
// below the cut the angle is pruned, otherwise it is listed at the end of the match's angle list (n_eval[b] of them)
// for k_sweep_bound<BOUND_SELECT>, which bounds it and keeps it by the same rule.  pruned_total += the angles left
// out here.  One CTA per match.
__global__ void __launch_bounds__(256)
    k_prune_select(const int32_t *__restrict__ sums, const double *__restrict__ ubr, const double *__restrict__ gub,
                   const double *__restrict__ centers, const int32_t *__restrict__ flags, b2s_matcher_params p,
                   b2s_search s, int n, int nx, int ny, int na, int32_t *__restrict__ angles,
                   int32_t *__restrict__ n_angles, uint8_t *__restrict__ keep, int32_t *__restrict__ n_eval,
                   double *__restrict__ cuts, unsigned long long *__restrict__ pruned_total) {
  const int b = blockIdx.x;
  const int f = flags[b];
  if ((f & 2) || !(f & 1)) {  // n_angles[b] is still 0, keep[b] all ones
    if (threadIdx.x == 0) n_eval[b] = 0;
    return;
  }
  __shared__ int32_t s_probe[PRUNE_PROBE];
  __shared__ double s_red[256];
  __shared__ float s_apf[PRUNE_MAX_ANGLES];
  __shared__ float s_fmax[256 / 32];
  __shared__ int s_cnt, s_ev;
  const int T = n_angles[b], ncell = nx * ny, ng = (na + BOUND_GROUP - 1) / BOUND_GROUP;
  if (threadIdx.x < T) s_probe[threadIdx.x] = angles[(size_t)b * na + threadIdx.x];
  if (threadIdx.x == 0) s_cnt = s_ev = 0;
  const bool pen = s.do_penalize != 0;
  const double ch = centers[3 * b + 2];
  const double start_a = ch - s.angle_offset;
  const double D = (double)((uint32_t)n * (uint32_t)GRID_OCCUPIED);
  const float inv_d = (float)(1.0 / D);
  red_angle_factors(s_apf, na, 0, start_a, ch, D, pen, s, p);
  __syncthreads();
  // The largest float score, then the exact response of the candidates the pre-filter cannot rule out: their maximum
  // is the maximum over every probed candidate.  A thread holds at most 4 cells (ncell <= 32 x 32, SweepPlan::prune);
  // only threads with such a candidate evaluate any.
  const int32_t *bs = sums + (size_t)b * na * ncell;
  float fmax_own = -1.0f;
  bool amb_own = false;
  for (int c = threadIdx.x; c < ncell; c += blockDim.x) {
    const int iy = c / nx, ix = c % nx;
    const double y = -s.offset_y + (double)(uint32_t)iy * s.res_y, x = -s.offset_x + (double)(uint32_t)ix * s.res_x;
    const float dpf = red_dist_factor(x * x + y * y, p);
    for (int t = 0; t < T; t++) {
      const int k = s_probe[t];
      bool amb;
      fmax_own = fmaxf(fmax_own, red_fscore(__ldcg(bs + (size_t)k * ncell + c), s_apf[k], dpf, inv_d, pen, amb));
      amb_own |= amb;
    }
  }
  float fmax = fmax_own;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) fmax = fmaxf(fmax, __shfl_xor_sync(0xffffffffu, fmax, d));
  if ((threadIdx.x & 31) == 0) s_fmax[threadIdx.x >> 5] = fmax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 256 / 32; w++) fmax = fmaxf(fmax, s_fmax[w]);
  const float thr = red_margin(fmax);
  double L = -1.0;
  for (int c = threadIdx.x; c < ncell && (fmax_own >= thr || amb_own); c += blockDim.x) {
    const int iy = c / nx, ix = c % nx;
    const double y = -s.offset_y + (double)(uint32_t)iy * s.res_y, x = -s.offset_x + (double)(uint32_t)ix * s.res_x;
    const double sq = x * x + y * y;
    const float dpf = red_dist_factor(sq, p);
    for (int t = 0; t < T; t++) {
      const int k = s_probe[t];
      const int32_t isum = __ldcg(bs + (size_t)k * ncell + c);
      bool amb;
      if (red_fscore(isum, s_apf[k], dpf, inv_d, pen, amb) < thr && !amb) continue;
      const double angle = start_a + (double)(uint32_t)k * s.angle_res;
      L = dmax(L, candidate_response(isum, n, pen, sq, angle, ch, p));
    }
  }
  s_red[threadIdx.x] = L;
  __syncthreads();
  for (int d = 128; d > 0; d >>= 1) {
    if (threadIdx.x < d) s_red[threadIdx.x] = dmax(s_red[threadIdx.x], s_red[threadIdx.x + d]);
    __syncthreads();
  }
  L = s_red[0];
  const bool all = !(L - 0.1 > 1.0e-6);
  const double cut = L - 0.1 - 1.0e-9;
  int pruned = 0;
  for (int k = threadIdx.x; k < na; k += blockDim.x) {
    if (keep[(size_t)b * na + k]) continue;  // probed
    const double u = ubr[(size_t)b * na + k];
    if (all || u >= cut) {
      angles[(size_t)b * na + atomicAdd(&s_cnt, 1)] = k;
      keep[(size_t)b * na + k] = 1;
    } else if (isnan(u) && gub[(size_t)b * ng + k / BOUND_GROUP] >= cut) {
      angles[(size_t)b * na + na - 1 - atomicAdd(&s_ev, 1)] = k;
    } else {
      pruned++;
    }
  }
  if (pruned) atomicAdd(pruned_total, (unsigned long long)pruned);
  __syncthreads();
  if (threadIdx.x == 0) {
    n_angles[b] = s_cnt;
    n_eval[b] = s_ev;
    cuts[b] = cut;
  }
}

// The empty windows of the last pruned sweep, counted when they are asked for (b2s_matcher_last_stats): every
// (beam, angle) pair of every match the window kernel swept, placed by win_origin_class as the lists would place it.
// The pruned sweep itself places only the beams of the angles it bounds one by one.  One block per (match, chunk of
// OFF_CHUNK angles).
__global__ void __launch_bounds__(256)
    k_count_empty(const double *__restrict__ local, const double *__restrict__ grid_off,
                  const double *__restrict__ centers, const int32_t *__restrict__ bases,
                  const int32_t *__restrict__ flags, const uint16_t *__restrict__ sat_all, int sbx, int sby,
                  double angle_offset, double angle_res, int na, int n, int ncell, int width_step, int data_size,
                  double scale, int rows_total, int cols_total, int height, int nx, int ny,
                  unsigned long long *__restrict__ stats) {
  const int chunks = (na + OFF_CHUNK - 1) / OFF_CHUNK;
  const int b = blockIdx.x / chunks, k0 = (blockIdx.x % chunks) * OFF_CHUNK;
  const int f = flags[b];
  if ((f & 2) || !(f & 1)) return;
  const int SW = sbx + 1;
  const uint16_t *sat = sat_all + (size_t)b * (((sby + 1) * SW + 7) & ~7);
  const WinGeom G = win_geom(grid_off[2 * b], grid_off[2 * b + 1], scale, bases[(size_t)b * ncell], 1, rows_total,
                             cols_total, width_step, data_size, height, nx, ny, 1, 1, 0);
  const double center = centers[(size_t)b * 3 + 2];
  unsigned long long cnt = 0;
  for (int k = k0; k < min(k0 + OFF_CHUNK, na); k++) {
    const double ang = win_angle(center, angle_offset, angle_res, k);
    const double c = cos(ang), sn = sin(ang);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      int32_t a;
      bool empty;
      win_origin_class(local[((size_t)b * n + i) * 2], local[((size_t)b * n + i) * 2 + 1], c, sn, G, true, sat, SW, a, empty);
      cnt += empty;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(stats, cnt);
}

__global__ void __launch_bounds__(RED_THREADS, 2) k_reduce(ReduceArgs A) {
  const int b = blockIdx.x;
  const int32_t *sums = A.sums;
  const double *__restrict__ centers = A.centers;
  const int32_t *__restrict__ flags = A.flags;
  const b2s_matcher_params &p = A.p;
  const b2s_search &s = A.s;
  const b2s_grid_info &g = A.g;
  const double scale = A.scale;
  const int n = A.n, nx = A.nx, ny = A.ny, na = A.na;
  double *__restrict__ probs_all = A.probs_all;
  b2s_match_result *__restrict__ results = A.results;
  const int k_first = A.k_first;
  const ReducePhase phase = A.phase;
  double *__restrict__ part_best = A.part_best;
  const double *__restrict__ glob_best = A.glob_best;
  double *__restrict__ tie_out = A.tie_out;
  const double *__restrict__ tie_in = A.tie_in;
  const int tid = threadIdx.x;
  const int ncell = nx * ny;
  b2s_match_result *res = results + b;
  if (flags[b] & 2) {
    if (tid == 0) res->status = B2S_ERR_OUT_OF_RANGE;
    return;
  }
  const int32_t *bs = sums + (size_t)b * na * ncell;
  const double cx = centers[3 * b], cy = centers[3 * b + 1], ch = centers[3 * b + 2];
  const double start_x = -s.offset_x, start_y = -s.offset_y, start_a = ch - s.angle_offset;
  const int pstep = (g.search_side + 7) & ~7;
  double *probs = probs_all + (size_t)b * pstep * g.search_side;
  const double pox = cx - s.offset_x, poy = cy - s.offset_y;  // Mapper.cpp:332-333
  const bool pen = s.do_penalize != 0;

  __shared__ double red[8];
  __shared__ double cov_terms[4][RED_THREADS];  // also the scratch of the block-wide max reduction
  __shared__ float s_apf[1024];  // per-angle factor (anglePenalty / (N*100)) as float
  __shared__ int s_err, s_count;
  __shared__ int tie_idx[RED_MAX_TIES];
  __shared__ int sorted[RED_MAX_TIES];
  __shared__ double s_best;
  __shared__ double s_mean[3];
  __shared__ uint8_t s_keep[PRUNE_MAX_ANGLES];
  __shared__ uint16_t s_list[PRUNE_MAX_ANGLES];
  __shared__ int s_nk;
  // A pruned sweep (keep != nullptr, na <= PRUNE_MAX_ANGLES) swept only the angles of keep; the others read 0, so
  // none of their candidates is a cell maximum above 0 or a tie (k_prune_select skips angles only when best > 0.1),
  // and the passes below walk only the swept angles, ascending: s_list[0, nk).  Otherwise they walk 0 .. na-1.
  const bool masked = A.keep != nullptr;
  for (int k = tid; k < na && masked; k += RED_THREADS) s_keep[k] = A.keep[(size_t)b * na + k];
  if (tid == 0) { s_err = 0; s_count = 0; }
  if (!s.fine && phase <= REDUCE_SPLIT_BEST)
    for (int i = tid; i < pstep * g.search_side; i += RED_THREADS) probs[i] = 0.0;  // Clear (Mapper.cpp:329)

  // Float pre-filter.  The exact fp64 response (reference operation order, candidate_response) is only needed for
  // candidates that can be a maximum or a tie; a float score f = isum * w(c,k) with relative error < 3e-7 bounds it:
  // a candidate whose f is more than 2e-6 (relative) below the largest f of its cell / below (best - 1e-6) cannot
  // be the cell maximum / a tie.  Candidates whose unpenalised response is near the 1e-6 DoubleEqual threshold of
  // the penalty test (Mapper.cpp:399) are always evaluated exactly.
  const bool tab = na <= 1024;
  const double D = (double)((uint32_t)n * (uint32_t)GRID_OCCUPIED);
  const float inv_d = (float)(1.0 / D);
  if (tab) red_angle_factors(s_apf, na, k_first, start_a, ch, D, pen, s, p);
  __syncthreads();
  if (masked && tid < 32) {
    int cnt = 0;
    for (int k0 = 0; k0 < na; k0 += 32) {
      const bool kept = k0 + tid < na && s_keep[k0 + tid];
      const unsigned m = __ballot_sync(0xffffffffu, kept);
      if (kept) s_list[cnt + __popc(m & ((1u << tid) - 1u))] = (uint16_t)(k0 + tid);
      cnt += __popc(m);
    }
    if (tid == 0) s_nk = cnt;
  }
  __syncthreads();
  const int nk = masked ? s_nk : na;
  // visit(k, sum) for the candidates of cell c in the walk's angle order, RED_UNROLL loads in flight; instantiated
  // with and without the list, so that an unpruned walk carries no list lookup
  auto walk = [&](auto listed, int c, auto &&visit) {
    for (int j0 = 0; j0 < nk; j0 += RED_UNROLL) {
      int k[RED_UNROLL];
      int32_t v[RED_UNROLL];
#pragma unroll
      for (int u = 0; u < RED_UNROLL; u++) {
        if constexpr (decltype(listed)::value) k[u] = j0 + u < nk ? (int)s_list[j0 + u] : 0;
        else k[u] = j0 + u;
        v[u] = j0 + u < nk ? __ldcg(bs + (size_t)k[u] * ncell + c) : 0;
      }
#pragma unroll
      for (int u = 0; u < RED_UNROLL; u++)
        if (j0 + u < nk) visit(k[u], v[u]);
    }
  };
  auto walk_cell = [&](int c, auto &&visit) {
    if (masked) walk(std::true_type{}, c, visit);
    else walk(std::false_type{}, c, visit);
  };

  // ---- pass 1: best response + per-cell maxima (Mapper.cpp:430-451); one thread per (x,y) cell ----
  // One read of the cell's nA sums: the running float maximum remembers its angle and whether any OTHER candidate
  // came within the filter margin of it; if none did, the exact maximum is at that angle and needs one fp64
  // evaluation, otherwise (near-ties, e.g. equal sums under the clamped penalty) the row is re-read and every
  // candidate inside the margin is evaluated exactly.
  double best = -1.0;
  float fmax0 = 0.0f, fmax1 = 0.0f;  // float maxima of this thread's first two cells, kept for pass 2
  bool known0 = false, known1 = false;
  for (int c = tid; c < ncell && phase <= REDUCE_SPLIT_BEST; c += RED_THREADS) {
    const int iy = c / nx, ix = c % nx;
    const double y = start_y + (double)(uint32_t)iy * s.res_y, x = start_x + (double)(uint32_t)ix * s.res_x;
    const double sq = x * x + y * y;
    double cell_best = -1.0;
    if (tab) {
      const float dpf = red_dist_factor(sq, p);
      float fmax = -1.0f;
      int kmax = 0;
      int32_t vmax = 0;
      bool near = false, any_amb = false;
      walk_cell(c, [&](int k, int32_t v) {
        bool amb;
        const float f = red_fscore(v, s_apf[k], dpf, inv_d, pen, amb);
        any_amb |= amb;
        if (f > fmax) {
          near = fmax >= red_margin(f);  // the old maximum (and only it or its own near ones) may still be near
          fmax = f; kmax = k; vmax = v;
        } else if (f >= red_margin(fmax)) {
          near = true;
        }
      });
      if (c == tid) { fmax0 = fmax; known0 = !any_amb; }
      else if (c == tid + RED_THREADS) { fmax1 = fmax; known1 = !any_amb; }
      if (!near && !any_amb) {
        const double angle = start_a + (double)(uint32_t)(k_first + kmax) * s.angle_res;
        cell_best = candidate_response(vmax, n, pen, sq, angle, ch, p);
      } else if (fmax == 0.0f && !any_amb) {
        cell_best = 0.0;  // every sum is 0: response 0 / D, never penalised (Mapper.cpp:399)
      } else {
        const float thr = red_margin(fmax);
        walk_cell(c, [&](int k, int32_t v) {
          bool amb;
          const float f = red_fscore(v, s_apf[k], dpf, inv_d, pen, amb);
          if (f >= thr || amb) {
            const double angle = start_a + (double)(uint32_t)(k_first + k) * s.angle_res;
            cell_best = dmax(cell_best, candidate_response(v, n, pen, sq, angle, ch, p));
          }
        });
      }
    } else {
      for (int k = 0; k < na; k++) {  // not pruned (masked needs tab)
        const double angle = start_a + (double)(uint32_t)(k_first + k) * s.angle_res;
        cell_best = dmax(cell_best, candidate_response(__ldcg(bs + (size_t)k * ncell + c), n, pen, sq, angle, ch, p));
      }
    }
    best = dmax(best, cell_best);
    if (!s.fine) {
      const int32_t px = world_to_grid_1(cx + x, pox, scale), py = world_to_grid_1(cy + y, poy, scale);
      if (!(px >= 0 && px < g.search_side && py >= 0 && py < g.search_side)) {
        s_err = 1;  // GetDataPointer -> GridIndex throws (Karto.h:4553-4557)
      } else {
        // distinct candidates can share a probs cell only on degenerate lattices; max is order-free
        unsigned long long *pp = reinterpret_cast<unsigned long long *>(probs + px + (size_t)py * pstep);
        atomicMax(pp, (unsigned long long)__double_as_longlong(dmax(cell_best, 0.0)));
      }
    }
  }
  cov_terms[0][tid] = best;
  __syncthreads();
  for (int d = RED_THREADS / 2; d > 0; d >>= 1) {
    if (tid < d) cov_terms[0][tid] = dmax(cov_terms[0][tid], cov_terms[0][tid + d]);
    __syncthreads();
  }
  if (tid == 0) s_best = phase <= REDUCE_SPLIT_BEST ? cov_terms[0][0] : glob_best[b];
  __syncthreads();
  best = s_best;
  if (s_err) {
    if (tid == 0) res->status = B2S_ERR_OUT_OF_RANGE;
    return;
  }
  if (phase == REDUCE_SPLIT_BEST) {  // split sweep, phase 1: this angle subset's best (the per-cell maxima are in `probs`)
    if (tid == 0) { part_best[b] = best; res->status = B2S_OK; }
    return;
  }

  // ---- pass 2: poses tied with the best (Mapper.cpp:455-487) ----
  double ax = 0, ay = 0, tx = 0, ty = 0;
  const float tie_thr = (float)((best - KT_TOLERANCE) * (1.0 - 1.0e-6)) - 1.0e-9f;
  for (int c = tid; c < ncell && phase != REDUCE_SPLIT_FINISH; c += RED_THREADS) {
    if (c == tid && known0 && fmax0 < tie_thr) continue;  // no candidate of this cell can tie (pass 1's maximum)
    if (c == tid + RED_THREADS && known1 && fmax1 < tie_thr) continue;
    const int iy = c / nx, ix = c % nx;
    const double y = start_y + (double)(uint32_t)iy * s.res_y, x = start_x + (double)(uint32_t)ix * s.res_x;
    const double sq = x * x + y * y;
    const float dpf = red_dist_factor(sq, p);
    walk_cell(c, [&](int k, int32_t v) {
      if (tab) {
        bool amb;
        const float f = red_fscore(v, s_apf[k], dpf, inv_d, pen, amb);
        if (f < tie_thr && !amb) return;
      }
      const double angle = start_a + (double)(uint32_t)(k_first + k) * s.angle_res;
      const double r = candidate_response(v, n, pen, sq, angle, ch, p);
      if (double_equal(r, best)) {
        const double h = normalize_angle(angle);
        ax += cx + x; ay += cy + y; tx += cos(h); ty += sin(h);
        int slot = atomicAdd(&s_count, 1);
        if (slot < RED_MAX_TIES) tie_idx[slot] = c * na + k;
      }
    });
  }
  __syncthreads();
  if (phase == REDUCE_SPLIT_FINISH && tid == 0) s_count = (int)tie_in[5 * b + 4];
  __syncthreads();
  const int total = s_count;
  if (total == 0 && phase != REDUCE_SPLIT_TIES) {
    if (tid == 0) res->status = B2S_ERR_NO_BEST_POSE;  // Mapper.cpp:484-487
    return;
  }
  if (phase == REDUCE_SPLIT_FINISH) {
    if (tid == 0) { red[0] = tie_in[5 * b]; red[1] = tie_in[5 * b + 1]; red[2] = tie_in[5 * b + 2]; red[3] = tie_in[5 * b + 3]; }
    __syncthreads();
  } else if (total <= RED_MAX_TIES && phase == REDUCE_WHOLE) {
    // rank-sort the tie list by reference linear index, then one thread sums in that exact order
    for (int i = tid; i < total; i += RED_THREADS) {
      int v = tie_idx[i], rank = 0;
      for (int j = 0; j < total; j++) rank += (tie_idx[j] < v);
      sorted[rank] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double sx = 0, sy = 0, cxs = 0, sys = 0;
      for (int i = 0; i < total; i++) {
        int v = sorted[i];
        int c = v / na, k = v % na;
        int iy = c / nx, ix = c % nx;
        double y = start_y + (double)(uint32_t)iy * s.res_y, x = start_x + (double)(uint32_t)ix * s.res_x;
        double h = normalize_angle(start_a + (double)(uint32_t)(k_first + k) * s.angle_res);
        sx += cx + x; sy += cy + y; cxs += cos(h); sys += sin(h);
      }
      red[0] = sx; red[1] = sy; red[2] = cxs; red[3] = sys;
    }
    __syncthreads();
  } else {
    // fixed-order tree reduction (deterministic; differs from the sequential sum only in the last bits)
    cov_terms[0][tid] = ax; cov_terms[1][tid] = ay; cov_terms[2][tid] = tx; cov_terms[3][tid] = ty;
    __syncthreads();
    for (int d = RED_THREADS / 2; d > 0; d >>= 1) {
      if (tid < d)
        for (int q = 0; q < 4; q++) cov_terms[q][tid] += cov_terms[q][tid + d];
      __syncthreads();
    }
    if (tid == 0) { red[0] = cov_terms[0][0]; red[1] = cov_terms[1][0]; red[2] = cov_terms[2][0]; red[3] = cov_terms[3][0]; }
    __syncthreads();
  }
  if (phase == REDUCE_SPLIT_TIES) {  // split sweep, phase 2: this subset's tie sums {x, y, cos, sin, count}
    if (tid == 0) {
      tie_out[5 * b] = red[0]; tie_out[5 * b + 1] = red[1]; tie_out[5 * b + 2] = red[2]; tie_out[5 * b + 3] = red[3];
      tie_out[5 * b + 4] = (double)total;
    }
    return;
  }
  if (tid == 0) {
    double sx = red[0], sy = red[1], cxs = red[2], sys = red[3];
    sx /= total; sy /= total; cxs /= total; sys /= total;
    s_mean[0] = sx; s_mean[1] = sy; s_mean[2] = atan2(sys, cxs);
  }
  __syncthreads();
  const double mean0 = s_mean[0], mean1 = s_mean[1], mean2 = s_mean[2];

  // ---- covariance ----
  if (!s.fine) {
    // ComputePositionalCovariance (Mapper.cpp:535-630).  The four running sums are accumulated in the reference's
    // (y, x) order: the per-cell terms are produced in parallel (0.0 for cells the reference skips, which leaves a
    // sum unchanged), then four threads add one series each sequentially.
    double cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    const bool tiny = best < KT_TOLERANCE;
    double axx = 0, axy = 0, ayy = 0, norm = 0;  // live in threads 0..3 (one series each)
    const double dx = mean0 - cx, dy = mean1 - cy;
    if (!tiny) {
      for (int base = 0; base < ncell; base += RED_THREADS) {
        const int c = base + tid;
        double t0 = 0, t1 = 0, t2 = 0, t3 = 0;
        if (c < ncell) {
          const int iy = c / nx, ix = c % nx;
          const double y = start_y + (double)(uint32_t)iy * s.res_y, x = start_x + (double)(uint32_t)ix * s.res_x;
          const int32_t px = world_to_grid_1(cx + x, pox, scale), py = world_to_grid_1(cy + y, poy, scale);
          if (!(px >= 0 && px < g.search_side && py >= 0 && py < g.search_side)) {
            s_err = 1;
          } else {
            const double response = probs[px + (size_t)py * pstep];
            if (response >= (best - 0.1)) {
              t0 = response;
              t1 = ((x - dx) * (x - dx) * response);
              t2 = ((x - dx) * (y - dy) * response);
              t3 = ((y - dy) * (y - dy) * response);
            }
          }
        }
        cov_terms[0][tid] = t0; cov_terms[1][tid] = t1; cov_terms[2][tid] = t2; cov_terms[3][tid] = t3;
        __syncthreads();
        const int cnt = min(RED_THREADS, ncell - base);
        if (tid < 4) {
          double acc = tid == 0 ? norm : (tid == 1 ? axx : (tid == 2 ? axy : ayy));
          for (int i = 0; i < cnt; i++) acc += cov_terms[tid][i];
          if (tid == 0) norm = acc; else if (tid == 1) axx = acc; else if (tid == 2) axy = acc; else ayy = acc;
        }
        __syncthreads();
      }
      if (tid == 1) red[1] = axx;
      if (tid == 2) red[2] = axy;
      if (tid == 3) red[3] = ayy;
      __syncthreads();
    }
    if (s_err) {
      if (tid == 0) res->status = B2S_ERR_OUT_OF_RANGE;
      return;
    }
    if (tid != 0) return;
    if (tiny) {
      cov[0] = MAX_VARIANCE; cov[4] = MAX_VARIANCE;
      cov[8] = 4 * (s.angle_res * s.angle_res);
    } else {
      axx = red[1]; axy = red[2]; ayy = red[3];
      if (norm > KT_TOLERANCE) {
        double vxx = axx / norm, vxy = axy / norm, vyy = ayy / norm;
        const double vthth = 4 * (s.angle_res * s.angle_res);
        vxx = dmax(vxx, 0.1 * (s.res_x * s.res_x));
        vyy = dmax(vyy, 0.1 * (s.res_y * s.res_y));
        const double mult = 1.0 / best;
        cov[0] = vxx * mult; cov[1] = vxy * mult; cov[3] = vxy * mult; cov[4] = vyy * mult; cov[8] = vthth;
      }
      if (double_equal(cov[0], 0.0)) cov[0] = MAX_VARIANCE;
      if (double_equal(cov[4], 0.0)) cov[4] = MAX_VARIANCE;
    }
    for (int i = 0; i < 9; i++) res->cov[i] = cov[i];
  }
  if (tid != 0) return;
  res->pose[0] = mean0; res->pose[1] = mean1; res->pose[2] = mean2;
  // un-clamped best goes through `response` for k_angular_cov; it clamps afterwards.  Coarse: clamp here.
  res->response = s.fine ? best : (best > 1.0 ? 1.0 : best);  // Mapper.cpp:514-517
  res->status = B2S_OK;
  res->tie_count = total;
}

// ----------------------------------------------------------------------------------------------
// k_angular_cov: ComputeAngularCovariance (Mapper.cpp:641-692).  One CTA per match; warps over angles,
// lanes over beams (GetResponse at the best cell), then thread 0 accumulates in angle order.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_angular_cov(const uint8_t *__restrict__ grids, size_t grid_pitch, b2s_grid_info g,
                  const double *__restrict__ grid_off, const int32_t *__restrict__ lut,
                  const double *__restrict__ centers, b2s_search s, double scale, int n, int na,
                  b2s_match_result *__restrict__ results) {
  const int b = blockIdx.x;
  b2s_match_result *res = results + b;
  if (res->status != B2S_OK) return;
  extern __shared__ double s_resp[];  // [na]
  __shared__ int32_t s_base;
  __shared__ int s_bad;
  const double best = res->response;
  if (threadIdx.x == 0) {
    int32_t gx = world_to_grid_1(res->pose[0], grid_off[2 * b], scale) + g.roi_x;
    int32_t gy = world_to_grid_1(res->pose[1], grid_off[2 * b + 1], scale) + g.roi_y;
    s_bad = !(gx >= 0 && gx < g.width && gy >= 0 && gy < g.height);
    s_base = gx + gy * g.width_step;
  }
  __syncthreads();
  if (s_bad) {
    if (threadIdx.x == 0) res->status = B2S_ERR_OUT_OF_RANGE;
    return;
  }
  const uint8_t *grid = grids + (size_t)b * grid_pitch;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int k = warp; k < na; k += nw) {
    const int32_t *offs = lut + ((size_t)b * na + k) * n;
    int32_t sum = 0;
    for (int i = lane; i < n; i += 32) {
      int32_t o = offs[i];
      if (o == INVALID_SCAN) continue;
      int32_t idx = (int32_t)((uint32_t)s_base + (uint32_t)o);
      if (idx >= 0 && idx < g.data_size) sum += grid[idx];
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    if (lane == 0) {
      double r = (double)sum;
      r /= (double)((uint32_t)n * (uint32_t)GRID_OCCUPIED);
      s_resp[k] = r;
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double ch = centers[3 * b + 2];
  const double best_angle = normalize_angle_difference(res->pose[2], ch);
  const double start = ch - s.angle_offset;
  double norm = 0.0, acc = 0.0;
  for (int k = 0; k < na; k++) {
    const double angle = start + (double)(uint32_t)k * s.angle_res;
    const double response = s_resp[k];
    if (response >= (best - 0.1)) {
      norm += response;
      acc += ((angle - best_angle) * (angle - best_angle) * response);
    }
  }
  if (norm > KT_TOLERANCE) {
    if (acc < KT_TOLERANCE) acc = s.angle_res * s.angle_res;
    acc /= norm;
  } else {
    acc = 1000 * (s.angle_res * s.angle_res);
  }
  res->cov[8] = acc;
  if (best > 1.0) res->response = 1.0;
}

// fine-stage search centre = coarse mean (Mapper.cpp:278): copy result poses into the centre array
__global__ void k_results_to_centers(const b2s_match_result *__restrict__ results, double *__restrict__ centers,
                                     int batch) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  centers[3 * b] = results[b].pose[0];
  centers[3 * b + 1] = results[b].pose[1];
  centers[3 * b + 2] = results[b].pose[2];
}

// split sweep: per-match status out of / back into the result records (all-reduced with MAX between the phases)
__global__ void k_status_pack(const b2s_match_result *__restrict__ results, int32_t *__restrict__ st, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < batch) st[b] = results[b].status;
}
__global__ void k_status_apply(b2s_match_result *__restrict__ results, const int32_t *__restrict__ st, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < batch && st[b] != 0) results[b].status = st[b];  // a rank saw an out-of-range candidate: the reference throws
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------

static b2s_status layout_from_params(const b2s_matcher_params *p, b2s_grid_info *g) {
  if (p->resolution <= 0 || p->search_size <= 0 || p->smear_deviation < 0 || p->range_threshold <= 0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "ScanMatcher::Create: invalid parameters");
  *g = grid_layout(*p);
  double resolution = 1.0 / (1.0 / p->resolution);
  double min_dev = 0.5 * resolution, max_dev = 10 * resolution;  // Mapper.h:1041-1053 throws
  if (!(p->smear_deviation >= min_dev && p->smear_deviation <= max_dev))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "Mapper Error: smear deviation must be within [0.5, 10] x resolution");
  return B2S_OK;
}

// Between a b2s_matcher_correlate_scan_begin and its _end the handle's state must not change.
static b2s_status refuse_if_pending(const b2s_matcher *m) {
  if (m && m->pending) B2S_FAIL(B2S_ERR_BAD_STATE, "a b2s_matcher_correlate_scan_begin awaits its _end: the handle cannot change state in between");
  return B2S_OK;
}
static b2s_status require_scans_and_grids(const b2s_matcher *m) {
  if (!m->scans_set || !m->grids_set) B2S_FAIL(B2S_ERR_BAD_STATE, "scans and grids must be set first");
  return B2S_OK;
}

// last_ms from the events of the last sweep: lists, sweep, fp64 tail (a span whose events are not complete keeps its value)
static void read_sweep_ms(b2s_matcher *m) {
  for (int i = 0; i < 3; i++) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, m->ev[i], m->ev[i + 1]) == cudaSuccess) m->last_ms[i] = ms;
  }
}

static b2s_status run_correlate(b2s_matcher *m, const b2s_search *s, int k_first = 0, int na_override = -1,
                                ReducePhase phase = REDUCE_WHOLE);
static b2s_status launch_window(b2s_matcher *m, const SweepPlan &pl, const int32_t *angles);
static b2s_status count_empty(b2s_matcher *m);
static b2s_status launch_lists(b2s_matcher *m, const SweepPlan &pl, const b2s_search &s, int k_first, int listed_chunks,
                               bool count_empty);

// (re)build the per-match block summed-area tables after the grids changed
static b2s_status build_sat(b2s_matcher *m) {
  const size_t sm = sizeof(uint32_t) * (size_t)(m->sbx + 1) * (m->sby + 1);
  m->sat_valid = false;
  if (sm > LIST_SMEM_MAX || (m->g.width_step % 4) != 0 || (long long)m->sbx * m->sby >= 65535) return B2S_OK;  // no skipping
  if (sm > 16 * 1024) B2S_CUDA_CHECK(raise_dyn_smem(k_grid_sat, sm));
  k_grid_sat<<<m->batch, 256, sm, m->stream>>>(m->d_grids, m->grid_pitch, m->g.width_step, m->g.height, m->sbx, m->sby, m->d_sat);
  B2S_CUDA_CHECK(cudaGetLastError());
  m->sat_valid = true;
  return B2S_OK;
}

// (re)build the per-match pooled grids of the angle-pruning bound after the grids changed (the ones that fit)
static b2s_status build_pool(b2s_matcher *m) {
  for (int i = 0; i < 2; i++) {
    const PoolLayout &l = m->pool[i];
    if (!l.fits) continue;
    auto kern = i ? k_grid_pool<7> : k_grid_pool<4>;
    kern<<<dim3((unsigned)ceil_div(l.plane / 4, 256), grid_rows(m->batch)), 256, 0, m->stream>>>(
        m->d_grids, m->grid_pitch, m->g.data_size, m->g.width_step, l.lead, l.plane, m->d_pools[i], l.pitch, m->batch);
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

void b2s_matcher_destroy(b2s_matcher *m);
static b2s_status matcher_create_impl(const b2s_matcher_params *params, const b2s_laser *laser, int device, int max_batch,
                                      int max_base_scans, void *cuda_stream, b2s_matcher *m, const b2s_grid_info &g) {
  m->p = *params; m->l = *laser; m->g = g; m->device = device;
  m->max_batch = max_batch; m->max_base = max_base_scans; m->n = laser->n_readings;
  cudaDeviceProp prop;
  B2S_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  m->num_sms = prop.multiProcessorCount;
  m->smem_optin = (int)prop.sharedMemPerBlockOptin;
  cudaFuncAttributes fa;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_sweep_window<1, false, false>));
  m->win_static_smem = fa.sharedSizeBytes;
  B2S_CUDA_CHECK(cudaFuncGetAttributes(&fa, k_add_scan));
  m->add_static_smem = fa.sharedSizeBytes;
  B2S_CUDA_CHECK(m->stream.init(cuda_stream));
  for (auto &e : m->ev) B2S_CUDA_CHECK(e.create());
  // smear kernel on the host with glibc, exactly CorrelationGrid::CalculateKernel (Mapper.h:1032-1087)
  {
    int ks = g.kernel_size, half = ks / 2;
    std::vector<uint8_t> K((size_t)ks * ks);
    double resolution = 1.0 / (1.0 / params->resolution);
    for (int i = -half; i <= half; i++)
      for (int j = -half; j <= half; j++) {
        double d = hypot(i * resolution, j * resolution);
        double z = exp(-0.5 * pow(d / params->smear_deviation, 2));
        uint32_t kv = cast_u32(kround(z * GRID_OCCUPIED));
        K[(i + half) + ks * (j + half)] = (uint8_t)kv;
        if ((i != 0 || j != 0) && kv >= (uint32_t)GRID_OCCUPIED) m->smear_degenerate = true;
      }
    B2S_CUDA_CHECK(m->d_kernel.reserve(K.size()));
    B2S_CUDA_CHECK(cudaMemcpy(m->d_kernel, K.data(), K.size(), cudaMemcpyHostToDevice));
  }
  const size_t B = (size_t)max_batch, N = (size_t)std::max(m->n, 1);
  m->grid_pitch = (((size_t)g.data_size + 16) + 127) & ~(size_t)127;
  B2S_CUDA_CHECK(m->d_ranges.reserve(B * N));
  B2S_CUDA_CHECK(m->d_poses.reserve(B * 3));
  B2S_CUDA_CHECK(m->d_sensor.reserve(B * 3));
  B2S_CUDA_CHECK(m->d_pts.reserve(B * N * 2));
  B2S_CUDA_CHECK(m->d_local.reserve(B * N * 2));
  B2S_CUDA_CHECK(m->d_grids.reserve(B * m->grid_pitch));
  B2S_CUDA_CHECK(m->d_grid_off.reserve(B * 2));
  B2S_CUDA_CHECK(m->d_flags.reserve(B));
  B2S_CUDA_CHECK(m->d_probs.reserve(B * probs_len(g.search_side)));
  B2S_CUDA_CHECK(m->d_centers.reserve(B * 3));
  B2S_CUDA_CHECK(m->d_results.reserve(B));
  B2S_CUDA_CHECK(m->d_work.reserve(1));
  m->sbx = (g.width_step + 3) / 4;
  m->sby = (g.height + 3) / 4;
  B2S_CUDA_CHECK(m->d_sat.reserve(B * sat_stride(m->sbx, m->sby)));
  B2S_CUDA_CHECK(m->d_stats.reserve(2));
  for (int i = 0; i < 2; i++) {
    m->pool[i] = pool_layout(g, i ? 7 : 4, m->smem_optin, m->win_static_smem);
    if (m->pool[i].fits) B2S_CUDA_CHECK(m->d_pools[i].reserve(B * m->pool[i].pitch));
  }
  B2S_CUDA_CHECK(m->d_part_best.reserve(B));
  B2S_CUDA_CHECK(m->d_glob_best.reserve(B));
  B2S_CUDA_CHECK(m->d_tie.reserve(B * 5));
  B2S_CUDA_CHECK(m->d_status.reserve(B));
  B2S_CUDA_CHECK(m->h_results.reserve(B));
  B2S_CUDA_CHECK(m->h_stats.reserve(2));
  m->h_stats[0] = m->h_stats[1] = 0;
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_grids, 0, B * m->grid_pitch, m->stream));
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_results, 0, B * sizeof(b2s_match_result), m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_matcher_create(const b2s_matcher_params *params, const b2s_laser *laser, int device, int max_batch,
                              int max_base_scans, void *cuda_stream, b2s_matcher **out) {
  if (!params || !laser || !out || max_batch <= 0 || laser->n_readings < 0 || max_base_scans < 0)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "b2s_matcher_create: null/negative argument");
  *out = nullptr;
  b2s_grid_info g;
  b2s_status st = layout_from_params(params, &g);
  if (st) return st;
  if ((st = open_device(device))) return st;
  std::unique_ptr<b2s_matcher, decltype(&b2s_matcher_destroy)> m(new (std::nothrow) b2s_matcher(), b2s_matcher_destroy);
  if (!m) B2S_FAIL(B2S_ERR_CUDA, "out of host memory");
  if ((st = matcher_create_impl(params, laser, device, max_batch, max_base_scans, cuda_stream, m.get(), g))) return st;
  *out = m.release();
  return B2S_OK;
}

void b2s_matcher_destroy(b2s_matcher *m) {
  if (!m) return;
  cudaSetDevice(m->device);
  cudaStreamSynchronize(m->stream);
  delete m;
}

b2s_status b2s_matcher_grid_info(const b2s_matcher *m, b2s_grid_info *out) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  *out = m->g;
  return B2S_OK;
}

b2s_status b2s_matcher_set_kernel(b2s_matcher *m, int which) {
  if (!m || which < 0 || which > 3) B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad kernel selector");
  m->force_kernel = which;
  return B2S_OK;
}

b2s_status b2s_matcher_sync(b2s_matcher *m) {
  if (!m) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null handle");
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_matcher_set_scans(b2s_matcher *m, int batch, const double *ranges, const double *poses) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !ranges || !poses) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (batch <= 0 || batch > m->max_batch) B2S_FAIL(B2S_ERR_TOO_LARGE, "batch exceeds the handle's max_batch");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  m->batch = batch;
  const size_t n = (size_t)m->n;
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_ranges, ranges, sizeof(double) * batch * n, cudaMemcpyHostToDevice, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_poses, poses, sizeof(double) * batch * 3, cudaMemcpyHostToDevice, m->stream));
  k_scan_points<<<batch, 256, 0, m->stream>>>(m->d_ranges, m->d_poses, m->l, m->d_sensor, m->d_pts, m->d_local, nullptr);
  B2S_CUDA_CHECK(cudaGetLastError());
  m->scans_set = true;
  m->grids_set = false;
  m->have_sweep = false;
  return B2S_OK;
}

// base_ranges != NULL: the base scans' readings come from the host; otherwise pool_rows ([batch * n_base], host) names
// rows of the handle's device-resident scan pool
static b2s_status add_scans_impl(b2s_matcher *m, int n_base, const double *base_ranges, const int32_t *pool_rows,
                                 const double *base_poses) {
  B2S_NVTX("K1 add_scans (rasterise + smear)");
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || n_base < 0 || (n_base > 0 && ((!base_ranges && !pool_rows) || !base_poses))) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (!m->scans_set) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_set_scans must precede b2s_matcher_add_scans");
  if (n_base > m->max_base) B2S_FAIL(B2S_ERR_TOO_LARGE, "n_base exceeds the handle's max_base_scans");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  const size_t n = (size_t)m->n;
  const double resolution = 1.0 / (1.0 / m->p.resolution);
  const double scale = 1.0 / m->p.resolution;  // CorrelationGrid ctor SetScale (Mapper.h:1020)
  k_grid_offsets<<<ceil_div(B, 128), 128, 0, m->stream>>>(m->d_sensor, m->d_grid_off, B, m->g.roi_w, m->g.roi_h,
                                                          resolution);
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_grids, 0, (size_t)B * m->grid_pitch, m->stream));  // Grid::Clear
  m->n_base = n_base;
  if (n_base > 0 && n > 0) {
    const size_t need = (size_t)B * n_base;
    B2S_CUDA_CHECK(m->d_base_ranges.reserve(need * n));
    B2S_CUDA_CHECK(m->d_base_poses.reserve(need * 3));
    B2S_CUDA_CHECK(m->d_base_pts.reserve(need * n * 2));
    B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_base_poses, base_poses, sizeof(double) * need * 3, cudaMemcpyHostToDevice, m->stream));
    if (base_ranges) {
      B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_base_ranges, base_ranges, sizeof(double) * need * n, cudaMemcpyHostToDevice, m->stream));
      k_scan_points<<<(unsigned)need, 256, 0, m->stream>>>(m->d_base_ranges, m->d_base_poses, m->l, nullptr, m->d_base_pts, nullptr, nullptr);
    } else {
      for (size_t i = 0; i < need; i++)
        if (pool_rows[i] < 0 || (size_t)pool_rows[i] >= m->pool_count) B2S_FAIL(B2S_ERR_OUT_OF_RANGE, "scan pool row out of range");
      B2S_CUDA_CHECK(m->d_base_src.reserve(need));
      B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_base_src, pool_rows, sizeof(int32_t) * need, cudaMemcpyHostToDevice, m->stream));
      k_scan_points<<<(unsigned)need, 256, 0, m->stream>>>(m->d_pool, m->d_base_poses, m->l, nullptr, m->d_base_pts, nullptr, m->d_base_src);
    }
    // k_add_scan stages a whole base scan in shared memory (25 bytes per beam).  Beyond the device's opt-in limit
    // (about 9 300 beams on an H100) the sequential kernel, exact for any beam count, builds the grids instead.
    const size_t smem = n * (2 * sizeof(double) + 2 * sizeof(int) + 1) + sizeof(int) + 16;
    const bool staged = !m->smear_degenerate && smem + m->add_static_smem <= (size_t)m->smem_optin;
    if (staged && smem > 16 * 1024) B2S_CUDA_CHECK(raise_dyn_smem(k_add_scan, smem));
    if (staged) {
      k_add_scan<<<(unsigned)need, 256, smem, m->stream>>>(m->d_base_pts, m->d_sensor, m->d_grid_off, m->d_grids,
                                                           m->grid_pitch, m->d_kernel, m->g, scale, (int)n, n_base);
    } else {
      AsyncBuf<uint8_t> scratch(m->stream);
      B2S_CUDA_CHECK(scratch.alloc((size_t)B * n));
      k_add_scans_seq<<<ceil_div(B, 32), 32, 0, m->stream>>>(m->d_base_pts, m->d_sensor, m->d_grid_off, m->d_grids,
                                                             m->grid_pitch, m->d_kernel, m->g, scale, (int)n, n_base,
                                                             B, scratch);
    }
    B2S_CUDA_CHECK(cudaGetLastError());
  }
  m->grids_set = true;
  m->grid_high_bytes = false;
  m->have_sweep = false;
  if (b2s_status st = build_pool(m)) return st;
  return build_sat(m);
}

b2s_status b2s_matcher_add_scans(b2s_matcher *m, int n_base, const double *base_ranges, const double *base_poses) {
  if (n_base > 0 && !base_ranges) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  return add_scans_impl(m, n_base, base_ranges, nullptr, base_poses);
}

// ---- scan pool: readings that serve as base scans of many matches (a mapper's running window, near chains, loop
// candidates) are uploaded once and referenced by row afterwards
b2s_status b2s_matcher_pool_append(b2s_matcher *m, const double *ranges, int32_t *out_row) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !ranges) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const size_t n = (size_t)std::max(m->l.n_readings, 1);
  if ((m->pool_count + 1) * n > m->d_pool.cap) {  // full: twice the rows (256 at first)
    Buf<double> fresh;
    B2S_CUDA_CHECK(fresh.reserve(std::max<size_t>(256, 2 * m->pool_count) * n));
    if (m->pool_count)
      B2S_CUDA_CHECK(cudaMemcpyAsync(fresh, m->d_pool, sizeof(double) * m->pool_count * n, cudaMemcpyDeviceToDevice, m->stream));
    B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->d_pool = std::move(fresh);  // the old pool is freed with `fresh`
  }
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_pool + m->pool_count * n, ranges, sizeof(double) * n, cudaMemcpyHostToDevice, m->stream));
  if (out_row) *out_row = (int32_t)m->pool_count;
  m->pool_count++;
  return B2S_OK;
}

int32_t b2s_matcher_pool_count(const b2s_matcher *m) { return m ? (int32_t)m->pool_count : 0; }

b2s_status b2s_matcher_add_scans_pool(b2s_matcher *m, int n_base, const int32_t *pool_rows, const double *base_poses) {
  if (n_base > 0 && !pool_rows) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  return add_scans_impl(m, n_base, nullptr, pool_rows, base_poses);
}

b2s_status b2s_matcher_set_grids(b2s_matcher *m, const uint8_t *grids, const double *offsets) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !grids || !offsets) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (!m->scans_set) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_set_scans must precede b2s_matcher_set_grids");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  m->grid_high_bytes = false;  // the reference's grids hold 0..100; anything above 127 needs the generic kernel
  for (size_t i = 0, e = (size_t)B * m->g.data_size; i < e; i++)
    if (grids[i] > 127) { m->grid_high_bytes = true; break; }
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_grids, 0, (size_t)B * m->grid_pitch, m->stream));
  B2S_CUDA_CHECK(cudaMemcpy2DAsync(m->d_grids, m->grid_pitch, grids, (size_t)m->g.data_size, (size_t)m->g.data_size, B,
                                   cudaMemcpyHostToDevice, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_grid_off, offsets, sizeof(double) * 2 * B, cudaMemcpyHostToDevice, m->stream));
  m->grids_set = true;
  m->have_sweep = false;
  if (b2s_status st = build_pool(m)) return st;
  return build_sat(m);
}

b2s_status b2s_matcher_get_grid(b2s_matcher *m, int b, uint8_t *out_bytes, double out_offset[2]) {
  if (!m || b < 0 || b >= m->batch || !m->grids_set) B2S_FAIL(B2S_ERR_BAD_STATE, "no grid for this match");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  if (out_bytes)
    B2S_CUDA_CHECK(cudaMemcpyAsync(out_bytes, m->d_grids + (size_t)b * m->grid_pitch, (size_t)m->g.data_size,
                                   cudaMemcpyDeviceToHost, m->stream));
  if (out_offset)
    B2S_CUDA_CHECK(cudaMemcpyAsync(out_offset, m->d_grid_off + 2 * b, 2 * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_matcher_get_point_readings(b2s_matcher *m, int b, double *out_xy) {
  if (!m || !out_xy || b < 0 || b >= m->batch || !m->scans_set) B2S_FAIL(B2S_ERR_BAD_STATE, "no scan for this match");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  B2S_CUDA_CHECK(cudaMemcpyAsync(out_xy, m->d_pts + (size_t)b * m->n * 2, sizeof(double) * 2 * m->n,
                                 cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_matcher_compute_offsets(b2s_matcher *m, int b, double angle_center, double angle_offset,
                                       double angle_res, int32_t *out, int32_t *out_n_angles) {
  if (!m || !out || b < 0 || b >= m->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad argument");
  if (b2s_status st = require_scans_and_grids(m)) return st;
  if (angle_res == 0.0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "angle resolution must be non-zero");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int na = n_steps(angle_offset, angle_res);
  const size_t n = (size_t)m->n;
  Buf<int32_t> tmp;
  B2S_CUDA_CHECK(tmp.reserve(na * n));
  // one-match launch on the slices of match b
  k_offsets<<<na, 256, 0, m->stream>>>(m->d_ranges + (size_t)b * n, m->d_local + (size_t)b * n * 2,
                                       m->d_grid_off + 2 * b, nullptr, 0, angle_center, 1, angle_offset, angle_res, na,
                                       (int)n, m->g.width_step, 1.0 / m->p.resolution, tmp, 0);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(out, tmp, sizeof(int32_t) * na * n, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  if (out_n_angles) *out_n_angles = na;
  return B2S_OK;
}

// Enqueue a CorrelateScan (centers H2D, lookup lists, sweep, reduce, results D2H into the handle's pinned buffer) on the
// handle's stream and return without waiting: a caller with two handles overlaps one batch's uploads and small kernels
// with the other batch's sweep.  b2s_matcher_correlate_scan_end waits and hands the results out.
b2s_status b2s_matcher_correlate_scan_begin(b2s_matcher *m, const double *centers, const b2s_search *search,
                                            const b2s_match_result *cov_in) {
  if (!m || !centers || !search) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (b2s_status st = require_scans_and_grids(m)) return st;
  if (search->fine && !cov_in) B2S_FAIL(B2S_ERR_BAD_PARAMS, "the fine stage needs the incoming covariances (rCovariance is IN/OUT)");
  if (m->pending) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_correlate_scan_begin while an earlier one awaits its _end");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_centers, centers, sizeof(double) * 3 * B, cudaMemcpyHostToDevice, m->stream));
  if (search->fine) {  // rCovariance is IN/OUT for the fine stage (Mapper.cpp:648)
    for (int b = 0; b < B; b++) m->h_results[b] = cov_in[b];
    B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_results, m->h_results, sizeof(b2s_match_result) * B, cudaMemcpyHostToDevice, m->stream));
  }
  b2s_status st = run_correlate(m, search);
  if (st) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_stats, m->d_stats, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
  m->pending = true;
  m->pending_batch = B;
  return B2S_OK;
}

b2s_status b2s_matcher_correlate_scan_end(b2s_matcher *m, b2s_match_result *results) {
  if (!m || !results) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (!m->pending) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_correlate_scan_end without a pending b2s_matcher_correlate_scan_begin");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->pending_batch;  // the batch the _begin enqueued
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  m->pending = false;
  std::memcpy(results, m->h_results, sizeof(b2s_match_result) * B);
  if (m->last_path == 2 && m->last.na > 0 && m->n > 0) m->last_empty_frac = (double)*m->h_stats / ((double)B * m->last.na * m->n);
  else m->last_empty_frac = 0.0;
  m->empty_pending = m->last_pruned && m->last_plan.skip_empty && m->n > 0;  // counted by last_stats
  m->last_pruned_frac = m->last_pruned ? (double)m->h_stats[1] / ((double)B * m->last.na) : 0.0;
  read_sweep_ms(m);
  return B2S_OK;
}

b2s_status b2s_matcher_correlate_scan(b2s_matcher *m, const double *centers, const b2s_search *search,
                                      b2s_match_result *results) {
  if (!results) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  b2s_status st = b2s_matcher_correlate_scan_begin(m, centers, search, results);
  if (st) return st;
  return b2s_matcher_correlate_scan_end(m, results);
}

b2s_status b2s_matcher_match_scan(b2s_matcher *m, int do_penalize, int do_refine, b2s_match_result *results) {
  B2S_NVTX("K1 MatchScan (coarse + fine)");
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !results) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (b2s_status st = require_scans_and_grids(m)) return st;
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  if (m->n == 0) {  // Mapper.cpp:199-209: no readings -> pose passthrough, maximum covariance
    std::vector<double> sp((size_t)3 * B);
    B2S_CUDA_CHECK(cudaMemcpyAsync(sp.data(), m->d_sensor, sizeof(double) * 3 * B, cudaMemcpyDeviceToHost, m->stream));
    B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    for (int b = 0; b < B; b++) {
      std::memset(&results[b], 0, sizeof(b2s_match_result));
      for (int i = 0; i < 3; i++) results[b].pose[i] = sp[3 * b + i];
      results[b].cov[0] = MAX_VARIANCE; results[b].cov[4] = MAX_VARIANCE;
      results[b].cov[8] = 4 * (m->p.coarse_angle_resolution * m->p.coarse_angle_resolution);
    }
    return B2S_OK;
  }
  const double resolution = 1.0 / (1.0 / m->p.resolution);
  b2s_search coarse;
  coarse.offset_x = 0.5 * ((double)m->g.search_side - 1) * resolution;  // Mapper.cpp:228-230
  coarse.offset_y = coarse.offset_x;
  coarse.res_x = 2 * resolution;  // Mapper.cpp:233-234
  coarse.res_y = 2 * resolution;
  coarse.angle_offset = m->p.coarse_search_angle_offset;
  coarse.angle_res = m->p.coarse_angle_resolution;
  coarse.do_penalize = do_penalize;
  coarse.fine = 0;
  // search centre = scan (sensor) pose (Mapper.cpp:237)
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_centers, m->d_sensor, sizeof(double) * 3 * B, cudaMemcpyDeviceToDevice, m->stream));
  b2s_status st = run_correlate(m, &coarse);
  if (st) return st;
  if (m->p.use_response_expansion) {  // Mapper.cpp:242-272 — applied to the matches whose response is ~0
    B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
    B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    std::vector<b2s_match_result> keep(m->h_results.p, m->h_results.p + B);
    std::vector<char> pending(B, 0);
    bool any = false;
    for (int b = 0; b < B; b++)
      if (keep[b].status == B2S_OK && double_equal(keep[b].response, 0.0)) { pending[b] = 1; any = true; }
    double new_off = m->p.coarse_search_angle_offset;
    for (int it = 0; it < 3 && any; it++) {
      new_off += 20 * 0.01745329251994329577;  // math::DegreesToRadians(20)
      b2s_search ex = coarse;
      ex.angle_offset = new_off;
      B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_centers, m->d_sensor, sizeof(double) * 3 * B, cudaMemcpyDeviceToDevice, m->stream));
      st = run_correlate(m, &ex);
      if (st) return st;
      B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
      B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
      any = false;
      for (int b = 0; b < B; b++) {
        if (!pending[b]) continue;
        keep[b] = m->h_results[b];
        if (keep[b].status != B2S_OK || !double_equal(keep[b].response, 0.0)) pending[b] = 0;
        else any = true;
      }
    }
    for (int b = 0; b < B; b++) m->h_results[b] = keep[b];
    B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_results, m->h_results, sizeof(b2s_match_result) * B, cudaMemcpyHostToDevice, m->stream));
  }
  if (do_refine) {  // Mapper.cpp:274-282
    b2s_search fine;
    fine.offset_x = coarse.res_x * 0.5;
    fine.offset_y = coarse.res_y * 0.5;
    fine.res_x = resolution;
    fine.res_y = resolution;
    fine.angle_offset = 0.5 * m->p.coarse_angle_resolution;
    fine.angle_res = m->p.fine_search_angle_offset;
    fine.do_penalize = do_penalize;
    fine.fine = 1;
    k_results_to_centers<<<ceil_div(B, 128), 128, 0, m->stream>>>(m->d_results, m->d_centers, B);
    st = run_correlate(m, &fine);
    if (st) return st;
  }
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  std::memcpy(results, m->h_results, sizeof(b2s_match_result) * B);
  return B2S_OK;
}

b2s_status b2s_matcher_match_scan_host(b2s_matcher *m, int batch, const double *ranges, const double *poses,
                                       int n_base, const double *base_ranges, const double *base_poses,
                                       int do_penalize, int do_refine, b2s_match_result *results) {
  b2s_status st = b2s_matcher_set_scans(m, batch, ranges, poses);
  if (st) return st;
  st = b2s_matcher_add_scans(m, n_base, base_ranges, base_poses);
  if (st) return st;
  return b2s_matcher_match_scan(m, do_penalize, do_refine, results);
}

/* ---- a CorrelateScan whose ANGLES are split over several GPUs (SURVEY.md §8(e)(ii)) ----
 * Every rank holds the same scans + grids and sweeps angle indices [k_first, k_first + k_count) of the search.
 * Between the three phases the caller all-reduces small host arrays (torch.distributed / NCCL):
 *   begin : out best[B] (MAX), per-cell maxima plane probs[B][probs_len] (MAX), status[B] (MAX)
 *   ties  : in global best; out tie sums {x, y, cos, sin, count}[B][5] (SUM)
 *   finish: in global best / tie sums / plane; out the same results as b2s_matcher_correlate_scan (coarse stage). */
b2s_status b2s_matcher_correlate_split_begin(b2s_matcher *m, const double *centers, const b2s_search *search, int k_first,
                                             int k_count, double *best, double *probs, int32_t *status) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !centers || !search || !best || !probs || !status || k_count < 0) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (search->fine) B2S_FAIL(B2S_ERR_BAD_PARAMS, "only the coarse stage (doingFineMatch = false) can be split");
  if (b2s_status st = require_scans_and_grids(m)) return st;
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  const size_t plen = probs_len(m->g.search_side);
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_centers, centers, sizeof(double) * 3 * B, cudaMemcpyHostToDevice, m->stream));
  b2s_status st = run_correlate(m, search, k_first, k_count, REDUCE_SPLIT_BEST);
  if (st) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(best, m->d_part_best, sizeof(double) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(probs, m->d_probs, sizeof(double) * plen * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  for (int b = 0; b < B; b++) status[b] = m->h_results[b].status;
  return B2S_OK;
}

static ReduceArgs reduce_args(b2s_matcher *m, const b2s_search &s, int nx, int ny, int na, int k_first, ReducePhase phase) {
  ReduceArgs A;
  A.sums = m->d_sums; A.centers = m->d_centers; A.flags = m->d_flags;
  A.p = m->p; A.s = s; A.g = m->g; A.scale = 1.0 / m->p.resolution;
  A.n = m->n; A.nx = nx; A.ny = ny; A.na = na;
  A.probs_all = m->d_probs; A.results = m->d_results;
  A.k_first = k_first; A.phase = phase;
  A.part_best = m->d_part_best; A.glob_best = m->d_glob_best; A.tie_out = m->d_tie; A.tie_in = m->d_tie;
  A.keep = nullptr;
  return A;
}

static b2s_status split_phase(b2s_matcher *m, ReducePhase phase) {
  k_reduce<<<m->batch, RED_THREADS, 0, m->stream>>>(reduce_args(m, m->last_search, m->last.nx, m->last.ny, m->last.na, m->last_k_first, phase));
  B2S_CUDA_CHECK(cudaGetLastError());
  return B2S_OK;
}

b2s_status b2s_matcher_correlate_split_ties(b2s_matcher *m, const double *global_best, double *tie_sums) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !global_best || !tie_sums) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (!m->have_sweep) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_correlate_split_begin must come first");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_glob_best, global_best, sizeof(double) * B, cudaMemcpyHostToDevice, m->stream));
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_tie, 0, sizeof(double) * 5 * B, m->stream));
  b2s_status st = split_phase(m, REDUCE_SPLIT_TIES);
  if (st) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(tie_sums, m->d_tie, sizeof(double) * 5 * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  return B2S_OK;
}

b2s_status b2s_matcher_correlate_split_finish(b2s_matcher *m, const double *global_best, const double *tie_sums,
                                              const double *probs, b2s_match_result *results) {
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m || !global_best || !tie_sums || !probs || !results) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (!m->have_sweep) B2S_FAIL(B2S_ERR_BAD_STATE, "b2s_matcher_correlate_split_begin must come first");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  const int B = m->batch;
  const size_t plen = probs_len(m->g.search_side);
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_glob_best, global_best, sizeof(double) * B, cudaMemcpyHostToDevice, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_tie, tie_sums, sizeof(double) * 5 * B, cudaMemcpyHostToDevice, m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_probs, probs, sizeof(double) * plen * B, cudaMemcpyHostToDevice, m->stream));
  b2s_status st = split_phase(m, REDUCE_SPLIT_FINISH);
  if (st) return st;
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  std::memcpy(results, m->h_results, sizeof(b2s_match_result) * B);
  return B2S_OK;
}

/* The same angle-split CorrelateScan with the collectives INSIDE the library (SURVEY.md §8(e)(ii); north_star: "a single
 * NCCL all-reduce on the per-scan best-score"): every rank holds the same scans + grids and calls this with its rank; the
 * angle steps are partitioned by rank, and between the three phases the library all-reduces device buffers on the
 * handle's stream through the caller's NCCL communicator — best response (MAX, B doubles), per-cell maxima plane (MAX,
 * B x probs_len doubles), status (MAX), tie sums (SUM, 5B doubles).  No host staging; results equal the single-GPU
 * b2s_matcher_correlate_scan on every rank. */
b2s_status b2s_matcher_correlate_scan_split(b2s_matcher *m, void *nccl_comm, int rank, int world, const double *centers,
                                            const b2s_search *search, b2s_match_result *results) {
  if (!m || !nccl_comm || !centers || !search || !results || world < 1 || rank < 0 || rank >= world)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null / bad argument");
  if (m->pending) B2S_FAIL(B2S_ERR_BAD_STATE, "a b2s_matcher_correlate_scan_begin awaits its _end");
  if (search->fine) B2S_FAIL(B2S_ERR_BAD_PARAMS, "only the coarse stage (doingFineMatch = false) can be split");
  if (b2s_status st = require_scans_and_grids(m)) return st;
  const NcclApi &nc = nccl_api();
  if (!nc.ok) B2S_FAIL(B2S_ERR_BAD_STATE, "libnccl.so.2 could not be loaded (dlopen)");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  for (auto &e : m->ev_split)
    if (!e) B2S_CUDA_CHECK(e.create());
  const int B = m->batch;
  const size_t plen = probs_len(m->g.search_side);
  const int na_full = n_steps(search->angle_offset, search->angle_res);
  const int base = na_full / world, extra = na_full % world;  // contiguous, balanced (parallel.shard_bounds)
  const int k_first = rank * base + std::min(rank, extra), k_count = base + (rank < extra ? 1 : 0);
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->d_centers, centers, sizeof(double) * 3 * B, cudaMemcpyHostToDevice, m->stream));
  b2s_status st = run_correlate(m, search, k_first, k_count, REDUCE_SPLIT_BEST);
  if (st) return st;
  k_status_pack<<<ceil_div(B, 128), 128, 0, m->stream>>>(m->d_results, m->d_status, B);
  auto check_nccl = [&](int rc, const char *what) -> b2s_status {
    if (rc == 0) return B2S_OK;
    set_last_error(std::string(what) + " failed: " + (nc.error_string ? nc.error_string(rc) : "NCCL error"));
    return B2S_ERR_CUDA;
  };
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[0], m->stream));
  if ((st = check_nccl(nc.all_reduce(m->d_part_best, m->d_glob_best, (size_t)B, NCCL_FLOAT64, NCCL_MAX, nccl_comm, m->stream), "ncclAllReduce(best)"))) return st;
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[1], m->stream));
  if ((st = check_nccl(nc.all_reduce(m->d_probs, m->d_probs, plen * B, NCCL_FLOAT64, NCCL_MAX, nccl_comm, m->stream), "ncclAllReduce(plane)"))) return st;
  if ((st = check_nccl(nc.all_reduce(m->d_status, m->d_status, (size_t)B, NCCL_INT32, NCCL_MAX, nccl_comm, m->stream), "ncclAllReduce(status)"))) return st;
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[2], m->stream));
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_tie, 0, sizeof(double) * 5 * B, m->stream));
  if ((st = split_phase(m, REDUCE_SPLIT_TIES))) return st;
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[3], m->stream));
  if ((st = check_nccl(nc.all_reduce(m->d_tie, m->d_tie, (size_t)5 * B, NCCL_FLOAT64, NCCL_SUM, nccl_comm, m->stream), "ncclAllReduce(ties)"))) return st;
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[4], m->stream));
  if ((st = split_phase(m, REDUCE_SPLIT_FINISH))) return st;
  k_status_apply<<<ceil_div(B, 128), 128, 0, m->stream>>>(m->d_results, m->d_status, B);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaEventRecord(m->ev_split[5], m->stream));
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_results, m->d_results, sizeof(b2s_match_result) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  std::memcpy(results, m->h_results, sizeof(b2s_match_result) * B);
  float ms = 0;
  if (cudaEventElapsedTime(&ms, m->ev_split[0], m->ev_split[1]) == cudaSuccess) m->last_split_ms[0] = ms;  // best
  if (cudaEventElapsedTime(&ms, m->ev_split[1], m->ev_split[2]) == cudaSuccess) m->last_split_ms[1] = ms;  // plane + status
  if (cudaEventElapsedTime(&ms, m->ev_split[3], m->ev_split[4]) == cudaSuccess) m->last_split_ms[2] = ms;  // tie sums
  if (cudaEventElapsedTime(&ms, m->ev_split[0], m->ev_split[5]) == cudaSuccess) m->last_split_ms[3] = ms;  // all phases after the sweep
  return B2S_OK;
}

/* ms of the last b2s_matcher_correlate_scan_split: all-reduce(best), all-reduce(plane + status), all-reduce(tie sums),
 * everything between the end of the local sweep and the final results */
b2s_status b2s_matcher_last_split_timing(b2s_matcher *m, double out[4]) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  for (int i = 0; i < 4; i++) out[i] = m->last_split_ms[i];
  return B2S_OK;
}

b2s_status b2s_matcher_get_response_sums(b2s_matcher *m, int b, int32_t *out, int32_t dims[3]) {
  if (!m || !out || b < 0 || b >= m->batch) B2S_FAIL(B2S_ERR_BAD_PARAMS, "bad argument");
  if (!m->have_sweep) B2S_FAIL(B2S_ERR_BAD_STATE, "no sweep has been run");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  if (m->last_pruned) {  // list and sweep every angle of the last search (its bases and grids are still resident; the
                         // lists of the angles it skipped were not built, or are an earlier search's)
    if (b2s_status st = launch_lists(m, m->last_plan, m->last_search, m->last_k_first, 0, false)) return st;
    if (b2s_status st = launch_window(m, m->last_plan, nullptr)) return st;
    m->last_pruned = false;
  }
  const int nx = m->last.nx, ny = m->last.ny, na = m->last.na;
  std::vector<int32_t> tmp((size_t)nx * ny * na);
  B2S_CUDA_CHECK(cudaMemcpyAsync(tmp.data(), m->d_sums + (size_t)b * nx * ny * na, sizeof(int32_t) * tmp.size(),
                                 cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  // device layout [k][iy][ix] -> reference loop order [iy][ix][k]
  for (int k = 0; k < na; k++)
    for (int c = 0; c < nx * ny; c++) out[(size_t)c * na + k] = tmp[(size_t)k * nx * ny + c];
  if (dims) { dims[0] = ny; dims[1] = nx; dims[2] = na; }
  return B2S_OK;
}

b2s_status b2s_matcher_last_stats(b2s_matcher *m, double out[4]) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (m->empty_pending && !m->pending) {
    // a pruned sweep does not place every (beam, angle) pair: count its empty windows now, from its inputs when they
    // are still resident (NaN once set_scans / add_scans / set_grids replaced them)
    m->empty_pending = false;
    m->last_empty_frac = NAN;
    if (m->have_sweep) {
      B2S_CUDA_CHECK(cudaSetDevice(m->device));
      if (b2s_status st = count_empty(m)) return st;
    }
  }
  out[0] = m->last_empty_frac;
  out[1] = (double)m->last_path;
  out[2] = (double)m->last.na * m->last.nx * m->last.ny;
  out[3] = (double)m->n;
  return B2S_OK;
}

b2s_status b2s_matcher_last_pruned_frac(b2s_matcher *m, double *out) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  *out = m->last_pruned_frac;
  return B2S_OK;
}

b2s_status b2s_matcher_last_prune_state(b2s_matcher *m, int32_t dims[2], double *ubr, double *gub, uint8_t *swept,
                                        double *cut) {
  if (!m || !dims) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (b2s_status st = refuse_if_pending(m)) return st;
  if (!m->have_sweep || !m->last_pruned)
    B2S_FAIL(B2S_ERR_BAD_STATE, "the last sweep was not pruned, its angles were swept since, or its inputs were replaced");
  const int B = m->last_batch, na = m->last.na, ng = ceil_div(na, BOUND_GROUP);
  const bool arrays = ubr || gub || swept || cut;
  const bool fits = dims[0] == B && dims[1] == na;
  dims[0] = B;
  dims[1] = na;
  if (!arrays) return B2S_OK;
  if (!fits) B2S_FAIL(B2S_ERR_BAD_PARAMS, "the arrays are not sized for the last sweep's matches and angles");
  B2S_CUDA_CHECK(cudaSetDevice(m->device));
  std::vector<int32_t> flags((size_t)B);
  B2S_CUDA_CHECK(cudaMemcpyAsync(flags.data(), m->d_flags, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, m->stream));
  if (ubr) B2S_CUDA_CHECK(cudaMemcpyAsync(ubr, m->d_ubr, sizeof(double) * B * na, cudaMemcpyDeviceToHost, m->stream));
  if (gub) B2S_CUDA_CHECK(cudaMemcpyAsync(gub, m->d_gub, sizeof(double) * B * ng, cudaMemcpyDeviceToHost, m->stream));
  if (swept) B2S_CUDA_CHECK(cudaMemcpyAsync(swept, m->d_keep, (size_t)B * na, cudaMemcpyDeviceToHost, m->stream));
  if (cut) B2S_CUDA_CHECK(cudaMemcpyAsync(cut, m->d_cuts, sizeof(double) * B, cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  // a match the generic kernel swept was never bounded: its rows of d_ubr and d_cuts are an earlier call's
  for (int b = 0; b < B; b++) {
    if (!((flags[b] & 2) || !(flags[b] & 1))) continue;
    if (ubr) std::fill(ubr + (size_t)b * na, ubr + (size_t)(b + 1) * na, (double)NAN);
    if (cut) cut[b] = NAN;
  }
  return B2S_OK;
}

b2s_status b2s_matcher_last_timing(b2s_matcher *m, double out[4]) {
  if (!m || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  if (m->have_sweep && !m->pending && cudaSetDevice(m->device) == cudaSuccess && cudaStreamSynchronize(m->stream) == cudaSuccess) {
    // the events of the LAST sweep (whichever entry point ran it: correlate_scan, match_scan's last stage, a split phase)
    read_sweep_ms(m);
    cudaGetLastError();
  }
  out[0] = m->last_ms[0]; out[1] = m->last_ms[1]; out[2] = m->last_ms[2]; out[3] = (double)m->last_path;
  return B2S_OK;
}

}  // extern "C"

namespace b2s {

// The window sweep of plan pl over the handle's lists; angles != nullptr: only the angles of the per-match lists
// d_angles / d_n_angles (a pruned sweep)
static b2s_status launch_window(b2s_matcher *m, const SweepPlan &pl, const int32_t *angles) {
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_work, 0, sizeof(int), m->stream));
  const size_t smem = angles ? pl.listed_smem : pl.win_smem;
  auto launch = [&](auto kern) -> b2s_status {
    B2S_CUDA_CHECK(raise_dyn_smem(kern, smem));
    kern<<<pl.ctas, WIN_THREADS, smem, m->stream>>>(m->d_grids, m->grid_pitch, m->g.data_size, pl.copy_bytes,
                                                    m->d_lists, m->d_counts, m->d_starts, m->d_flags, m->batch, m->n,
                                                    pl.na, pl.nx, pl.ny, m->g.width_step, m->d_sums, m->d_work,
                                                    pl.band_rows, pl.nbands, pl.band_bytes, pl.neg_bands, angles,
                                                    angles ? m->d_n_angles.p : nullptr, pl.acc_slots);
    B2S_CUDA_CHECK(cudaGetLastError());
    return B2S_OK;
  };
  if (angles)  // a pruned sweep: stride 1, one tile (SweepPlan::prune)
    return pl.gen ? launch(k_sweep_window<1, true, true>) : launch(k_sweep_window<1, false, true>);
  if (pl.stride == 2) return pl.gen ? launch(k_sweep_window<2, true, false>) : launch(k_sweep_window<2, false, false>);
  return pl.gen ? launch(k_sweep_window<1, true, false>) : launch(k_sweep_window<1, false, false>);
}

// The window lists of plan pl for search s: every angle (listed_chunks == 0), or only the angles of the per-match
// lists d_angles / d_n_angles of a pruned sweep, listed_chunks * OFF_CHUNK of them at most.  count_empty: add the
// empty windows dropped to d_stats[0].
static b2s_status launch_lists(b2s_matcher *m, const SweepPlan &pl, const b2s_search &s, int k_first, int listed_chunks,
                               bool count_empty) {
  const int na = pl.na, ncell = pl.nx * pl.ny;
  auto launch = [&](auto kern, int chunks) -> b2s_status {
    if (pl.osm > 16 * 1024)  // static + dynamic shared memory together must stay under the 48 KB default: opt in early
      B2S_CUDA_CHECK(raise_dyn_smem(kern, pl.osm));
    kern<<<m->batch * chunks, 256, pl.osm, m->stream>>>(
        m->d_ranges, m->d_local, m->d_grid_off, m->d_centers, m->d_bases, m->d_flags, s.angle_offset, s.angle_res, na,
        m->n, ncell, m->g.width_step, m->g.data_size, 1.0 / m->p.resolution, pl.rows_total, pl.tiles_x * 32,
        m->d_lists, m->d_counts, pl.skip_empty ? m->d_sat.p : nullptr, m->sbx, m->sby, m->g.height, pl.nx, pl.ny,
        count_empty ? m->d_stats.p : nullptr, pl.band_rows, pl.nbands, m->d_starts, pl.stride, k_first, pl.neg_bands,
        listed_chunks ? m->d_angles.p : nullptr, listed_chunks ? m->d_n_angles.p : nullptr, chunks);
    B2S_CUDA_CHECK(cudaGetLastError());
    return B2S_OK;
  };
  if (listed_chunks) return launch(k_offsets_sorted<true>, listed_chunks);
  return launch(k_offsets_sorted<false>, ceil_div(na, OFF_CHUNK));
}

// last_empty_frac of the last (pruned) sweep from its resident inputs: k_count_empty over every (beam, angle) pair
static b2s_status count_empty(b2s_matcher *m) {
  const SweepPlan &pl = m->last_plan;
  const b2s_search &s = m->last_search;
  const int B = m->batch, na = pl.na;
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_stats, 0, sizeof(unsigned long long), m->stream));
  k_count_empty<<<B * ceil_div(na, OFF_CHUNK), 256, 0, m->stream>>>(
      m->d_local, m->d_grid_off, m->d_centers, m->d_bases, m->d_flags, m->d_sat, m->sbx, m->sby, s.angle_offset,
      s.angle_res, na, m->n, pl.nx * pl.ny, m->g.width_step, m->g.data_size, 1.0 / m->p.resolution, pl.rows_total,
      pl.tiles_x * 32, m->g.height, pl.nx, pl.ny, m->d_stats);
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaMemcpyAsync(m->h_stats, m->d_stats, sizeof(unsigned long long), cudaMemcpyDeviceToHost, m->stream));
  B2S_CUDA_CHECK(cudaStreamSynchronize(m->stream));
  m->last_empty_frac = (double)*m->h_stats / ((double)B * na * m->n);
  return B2S_OK;
}

// k_sweep_bound in mode MODE: the group pass over the 7x7 image, or single angles over the 4x4 image and the SAT
template <int MODE>
static b2s_status launch_bound(b2s_matcher *m, const SweepPlan &pl, const b2s_search &s) {
  constexpr bool GRP = MODE == BOUND_GROUPS;
  const PoolLayout &l = m->pool[GRP];
  const int rows = GRP ? pl.group_rows : pl.bound_rows;
  const size_t smem = (GRP ? pl.group_smem : pl.bound_smem) + (size_t)rows * BOUND_ROW_BYTES;
  auto kern = (GRP ? pl.group_stage : pl.bound_stage) ? k_sweep_bound<true, MODE> : k_sweep_bound<false, MODE>;
  B2S_CUDA_CHECK(cudaMemsetAsync(m->d_work, 0, sizeof(int), m->stream));
  B2S_CUDA_CHECK(raise_dyn_smem(kern, smem));
  kern<<<pl.ctas, WIN_THREADS, smem, m->stream>>>(
      m->d_pools[GRP], l.pitch, l.bytes, l.plane, l.lead, m->d_local, m->d_grid_off, m->d_bases,
      !GRP && pl.skip_empty ? m->d_sat.p : nullptr, m->sbx, m->sby, m->g.height, pl.rows_total, pl.tiles_x * 32,
      1.0 / m->p.resolution, m->d_flags, m->d_centers, m->p, s, m->batch, m->n, pl.na, pl.nx, pl.ny, m->g.width_step,
      m->g.data_size, m->d_ubr, m->d_gub, m->d_angles, m->d_n_angles, m->d_keep, m->d_n_eval, m->d_cuts,
      m->d_stats.p + 1, m->d_bscratch, rows, m->d_work);
  B2S_CUDA_CHECK(cudaGetLastError());
  return B2S_OK;
}

// the response sweep of a pruned search: group bounds, then bounds, probe, select, sweep the selected angles
static b2s_status run_pruned(b2s_matcher *m, const SweepPlan &pl, const b2s_search &s, int k_first) {
  const int B = m->batch, na = pl.na;
  if (pl.group) {
    if (b2s_status st = launch_bound<BOUND_GROUPS>(m, pl, s)) return st;
  } else {  // every group unbounded (0x7f7f... is a double near 1.4e306): every angle is bounded one by one
    B2S_CUDA_CHECK(cudaMemsetAsync(m->d_gub, 0x7f, sizeof(double) * (size_t)B * ceil_div(na, BOUND_GROUP), m->stream));
  }
  if (b2s_status st = launch_bound<BOUND_PROBE>(m, pl, s)) return st;
  if (b2s_status st = launch_lists(m, pl, s, k_first, ceil_div(PRUNE_PROBE, OFF_CHUNK), false)) return st;
  if (b2s_status st = launch_window(m, pl, m->d_angles)) return st;
  k_prune_select<<<B, 256, 0, m->stream>>>(m->d_sums, m->d_ubr, m->d_gub, m->d_centers, m->d_flags, m->p, s, m->n,
                                           pl.nx, pl.ny, na, m->d_angles, m->d_n_angles, m->d_keep, m->d_n_eval,
                                           m->d_cuts, m->d_stats.p + 1);
  B2S_CUDA_CHECK(cudaGetLastError());
  if (b2s_status st = launch_bound<BOUND_SELECT>(m, pl, s)) return st;
  if (b2s_status st = launch_lists(m, pl, s, k_first, ceil_div(na, OFF_CHUNK), false)) return st;
  return launch_window(m, pl, m->d_angles);
}

// One CorrelateScan over the batch with centres already in d_centers.  Results stay in d_results.
static b2s_status run_correlate(b2s_matcher *m, const b2s_search *s, int k_first, int na_override, ReducePhase phase) {
  B2S_NVTX("K1 correlate (lists + sweep + tail)");
  const SweepPlan pl = plan_sweep(m->p, m->g, *s, m->n, m->batch, k_first, na_override, m->force_kernel, m->sat_valid,
                                  m->grid_high_bytes, m->sbx, m->sby, m->num_sms, m->smem_optin, m->win_static_smem);
  if (pl.status) B2S_FAIL(pl.status, pl.error);
  const int B = m->batch, n = m->n, nx = pl.nx, ny = pl.ny, na = pl.na, ncell = nx * ny;
  const double scale = 1.0 / m->p.resolution;
  const bool lists = pl.use_window && na > 0;
  B2S_CUDA_CHECK(m->d_sums.reserve((size_t)B * na * ncell));
  B2S_CUDA_CHECK(m->d_bases.reserve((size_t)B * ncell));
  if (pl.need_plain_lut) B2S_CUDA_CHECK(m->d_lut.reserve((size_t)B * na * std::max(n, 1)));
  if (lists) {
    B2S_CUDA_CHECK(m->d_lists.reserve((size_t)B * na * (n + LIST_PAD * pl.nbands)));
    B2S_CUDA_CHECK(m->d_counts.reserve((size_t)B * na * 8 * pl.nbands));
    B2S_CUDA_CHECK(m->d_starts.reserve((size_t)B * na * 8 * pl.nbands));
  }
  m->empty_pending = false;
  if (pl.prune) {
    B2S_CUDA_CHECK(m->d_ubr.reserve((size_t)B * na));
    B2S_CUDA_CHECK(m->d_gub.reserve((size_t)B * ceil_div(na, BOUND_GROUP)));
    B2S_CUDA_CHECK(m->d_n_eval.reserve((size_t)B));
    B2S_CUDA_CHECK(m->d_cuts.reserve((size_t)B));
    B2S_CUDA_CHECK(m->d_bscratch.reserve((size_t)B * (na + ceil_div(na, BOUND_GROUP))));
    B2S_CUDA_CHECK(m->d_angles.reserve((size_t)B * na));
    B2S_CUDA_CHECK(m->d_n_angles.reserve((size_t)B));
    B2S_CUDA_CHECK(m->d_keep.reserve((size_t)B * na));
  }

  // ---- candidate bases, lookup tables, window lists ----
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[0], m->stream));
  k_bases<<<B, 256, 0, m->stream>>>(m->d_centers, m->d_grid_off, *s, m->g, scale, nx, ny, m->d_bases, m->d_flags,
                                    std::max(pl.stride, 1));
  if (pl.need_plain_lut && na > 0)
    k_offsets<<<B * na, 256, 0, m->stream>>>(m->d_ranges, m->d_local, m->d_grid_off, m->d_centers, 3, 0.0, 0,
                                             s->angle_offset, s->angle_res, na, n, m->g.width_step, scale, m->d_lut, k_first);
  if (lists) {
    B2S_CUDA_CHECK(cudaMemsetAsync(m->d_stats, 0, 2 * sizeof(unsigned long long), m->stream));
    // a pruned sweep lists only the angles it sweeps, inside the sweep stage; its empty windows are counted on request
    if (!pl.prune)
      if (b2s_status st = launch_lists(m, pl, *s, k_first, 0, true)) return st;
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[1], m->stream));

  // ---- response sweep ----
  if (na == 0) {
    m->last_path = pl.use_window ? 2 : 1;  // empty angle subset of a split sweep: nothing to sweep
  } else if (pl.use_window) {
    // (A variant that ran each match's fp64 tail inside the sweep CTA right after its last tile — volume read back from
    // L2, no k_reduce pass — was built, parity-tested and measured SLOWER on cfg 2 (not re-measured on the H100): the
    // sweep kernel owns its SM, so the tail's serial stretches are no longer hidden by a second resident CTA as they are
    // in the stand-alone k_reduce.  Removed again; DESIGN.md §4.)
    if (pl.prune) {
      if (b2s_status st = run_pruned(m, pl, *s, k_first)) return st;
    } else {
      if (pl.nbands > 1)  // bands accumulate with RED.ADD
        B2S_CUDA_CHECK(cudaMemsetAsync(m->d_sums, 0, sizeof(int32_t) * (size_t)B * na * ncell, m->stream));
      if (b2s_status st = launch_window(m, pl, nullptr)) return st;
    }
    // matches whose lattice is not the regular raster (a centre exactly on a rounding tie) fall through;
    // they compute their lookup values on the fly (no table was materialised for them)
    // (a few CTAs per match that exit at once unless the lattice is irregular: the kernel loops over the cells)
    k_sweep_generic<<<dim3(4, grid_rows(B)), 256, 0, m->stream>>>(m->d_grids, m->grid_pitch, m->g.data_size, nullptr, m->d_bases,
                                                  m->d_flags, 1, n, na, ncell, m->d_sums, m->d_ranges, m->d_local,
                                                  m->d_grid_off, m->d_centers, s->angle_offset, s->angle_res,
                                                  m->g.width_step, scale, k_first, B);
    m->last_path = 2;
  } else {
    k_sweep_generic<<<dim3((unsigned)ceil_div(ncell, 8), grid_rows(B)), 256, 0, m->stream>>>(
        m->d_grids, m->grid_pitch, m->g.data_size, m->d_lut, m->d_bases, m->d_flags, 0, n, na, ncell, m->d_sums,
        m->d_ranges, m->d_local, m->d_grid_off, m->d_centers, s->angle_offset, s->angle_res, m->g.width_step, scale,
        k_first, B);
    m->last_path = 1;
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[2], m->stream));

  // ---- fp64 tail ----
  ReduceArgs ra = reduce_args(m, *s, nx, ny, na, k_first, phase);
  if (pl.prune) ra.keep = m->d_keep;
  k_reduce<<<B, RED_THREADS, 0, m->stream>>>(ra);
  if (s->fine) {  // plan_sweep refused angle counts whose responses do not fit in 48 KB
    // the kernel's own static shared memory comes on top: 48 KB of responses (6 144 angles) needs the opt-in
    if (sizeof(double) * (size_t)na > 16 * 1024) B2S_CUDA_CHECK(raise_dyn_smem(k_angular_cov, sizeof(double) * (size_t)na));
    k_angular_cov<<<B, 256, sizeof(double) * (size_t)na, m->stream>>>(m->d_grids, m->grid_pitch, m->g, m->d_grid_off,
                                                                      m->d_lut, m->d_centers, *s, scale, n, na,
                                                                      m->d_results);
  }
  B2S_CUDA_CHECK(cudaGetLastError());
  B2S_CUDA_CHECK(cudaEventRecord(m->ev[3], m->stream));
  m->last.nx = nx; m->last.ny = ny; m->last.na = na;
  m->last_plan = pl;
  m->last_pruned = pl.prune && na > 0;
  m->last_batch = B;
  m->last_search = *s;
  m->last_k_first = k_first;
  m->have_sweep = true;
  return B2S_OK;
}

}  // namespace b2s
