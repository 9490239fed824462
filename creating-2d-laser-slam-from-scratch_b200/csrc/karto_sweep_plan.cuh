// The host-side plan of one Karto correlative sweep (karto_matcher.cu, run_correlate): which sweep kernel runs, the
// candidate stride, the row-band geometry of the window kernel and the shared-memory sizes of the list and sweep stages,
// or the refusal of the search.  Pure arithmetic on the handle's geometry with no CUDA call, so that it can be checked
// on a machine without a GPU (tests/sweep_plan_check.cu).
//
// The kernels are correct only if these numbers are: the bands must cover every window origin row, and the staged image
// must hold every row a lane touches.  The constants below are the ones the kernels and the plan must agree on.
#pragma once

#include "common.cuh"

namespace b2s {

constexpr int WIN_THREADS = 512;
constexpr int WIN_GUARD = 128;          // zero bytes before and after the grid image in shared memory
constexpr int WIN_MAX_BANDS = 32;       // row bands a grid larger than shared memory is swept in
constexpr int LIST_PAD = 16;            // per-(match, angle) list capacity = n + LIST_PAD * nbands
constexpr int OFF_CHUNK = 16;           // angles per k_offsets_sorted block
constexpr int OFF_Q = 2;                              // angles classified per pass
constexpr int OFF_SMEM_PER_BEAM = 16 + 5 * OFF_Q;     // two doubles + OFF_Q x (origin int32 + class byte)
constexpr size_t LIST_SMEM_MAX = 200 * 1024;  // dynamic shared memory of the list stage and of the SAT build
constexpr int PRUNE_MIN_ANGLES = 32;    // fewer angles: the bound pass and the probe cost more than they save
constexpr int PRUNE_MAX_ANGLES = 1024;  // the select kernels and k_reduce's angle mask hold one entry per angle
constexpr int PRUNE_PROBE = 16;         // angles swept exactly to find the pruning threshold (one per sweep warp)
// consecutive angles the group pass of the bound takes at once: at cfg 2 a beam's window origin moves at most 2.42
// cells per axis over 3 angle steps, so the four origins lie in a 4 x 4 cell square and a 7 x 7 pooled image read at
// the square's low corner bounds all four (k_sweep_bound_group)
constexpr int BOUND_GROUP = 4;
constexpr int BOUND_SPREAD = 3;  // the origin spread per axis the 7 x 7 image covers: 7 = 4 + BOUND_SPREAD

// Work items of a pruned search's rounds.  A round of few units (at most `cap`, the shared-memory accumulators that
// fit) cuts each unit's `total` beams into `chunks` ranges on multiples of QUANTUM, so that every warp of the CTA gets
// about two items with at least MIN_BEAMS beams per range on average; the ranges' partial sums meet in the unit's
// accumulator.  A round of more units is one item per unit.  Two instances, below: k_sweep_window<LISTED>'s (a unit is
// a listed angle, its accumulator an ny x nx plane, acc_slots) and k_sweep_bound's (a unit is an angle or a group of
// BOUND_GROUP angles, its accumulator a u32 row of block sums, bound_rows / group_rows; 32: a warp's placement pass).
constexpr int WIN_CHUNK_MIN_BEAMS = 32;     // a window item costs ~250 instructions besides its beams
constexpr int BOUND_CHUNK_MIN_BEAMS = 128;  // a bound item costs the unit's sincos, shuffles and row adds besides its beams
constexpr int BOUND_ROW_BYTES = 64 * 4;     // one u32 per 4 x 4 block of the 32 x 32 candidate tile
template <int QUANTUM, int MIN_BEAMS>
__host__ __device__ inline int split_chunks(int units, int n, int warps, int cap) {
  static_assert(MIN_BEAMS % QUANTUM == 0, "a range of MIN_BEAMS beams is whole quanta");
  if (units <= 0 || units > cap) return 1;
  const int want = (2 * warps + units - 1) / units;
  const int most = n / MIN_BEAMS;
  return most < 2 ? 1 : (want < most ? want : most);
}
__host__ __device__ constexpr int log2_of(int v) { return v > 1 ? 1 + log2_of(v >> 1) : 0; }
// the beams [lo, hi) of range c of `chunks` of a unit of `total` beams
template <int QUANTUM>
__host__ __device__ inline void split_range(int total, int c, int chunks, int &lo, int &hi) {
  static_assert((QUANTUM & (QUANTUM - 1)) == 0, "a power of two: the quanta are a shift");
  const long long q = (total + QUANTUM - 1) >> log2_of(QUANTUM);
  lo = QUANTUM * (int)(q * c / chunks);
  hi = QUANTUM * (int)(q * (c + 1) / chunks);
  if ((total & (QUANTUM - 1)) && hi > total) hi = total;  // only a total of part quanta ends inside the last one
}
// the window's: an angle's beams are its groups I0 I1 I2 I3 E0 E1 E2 E3, each a multiple of 4 long; the mask tells the
// compiler so, and split_range's round-up and clamp vanish
__host__ __device__ inline int listed_chunks(int listed, int n, int warps, int slots) { return split_chunks<4, WIN_CHUNK_MIN_BEAMS>(listed, n, warps, slots); }
__host__ __device__ inline void chunk_range(int total, int c, int chunks, int &lo, int &hi) { split_range<4>(total & ~3, c, chunks, lo, hi); }
// the bound's
__host__ __device__ inline int bound_chunks(int units, int n, int warps, int rows) { return split_chunks<32, BOUND_CHUNK_MIN_BEAMS>(units, n, warps, rows); }
__host__ __device__ inline void bound_range(int n, int c, int chunks, int &lo, int &hi) { split_range<32>(n, c, chunks, lo, hi); }
// the part of each group g (count[g] beams) that lies in [lo, hi): beams off[g] .. off[g] + len[g] of the group
__host__ __device__ inline void chunk_groups(const int32_t *count, int lo, int hi, int (&off)[8], int (&len)[8]) {
  int p = 0;
#pragma unroll
  for (int g = 0; g < 8; g++) {
    const int s = lo > p ? lo - p : 0, e = hi - p < count[g] ? hi - p : count[g];
    off[g] = s;
    len[g] = e > s ? e - s : 0;
    p += count[g];
  }
}

// u16 entries per match of the block summed-area tables (k_grid_sat), padded to 16 bytes
inline size_t sat_stride(int sbx, int sby) { return (size_t)((((sbx + 1) * (sby + 1)) + 7) & ~7); }
// The K x K max-pooled grid (k_grid_pool) of one match, K = 4 for k_sweep_bound's single angles, K = 7 for its group
// pass: P[f] = max over dy, dx in [0, K) of grid[f + dy * width_step + dx] (0 outside the grid), for f from -lead on:
// 4 rows (a block whose corner lies above the grid still reaches it), 8 for K = 7 (a group's low corner lies up to
// BOUND_SPREAD rows and columns before any member's origin).  It is stored as four planes split by the residue of
// j = f + lead modulo 4: plane j & 3 byte j >> 2 holds P[f] (pool_index), each plane `plane` bytes long.  A beam's 8
// block corners of one block row are 4 apart in f, so they are 8 contiguous bytes of one plane, and the rows are
// width_step bytes apart in it (width_step % 8 == 0: one word alignment for all 8 rows).  Each plane ends with
// POOL_PAD or more zero bytes (P of indices past the grid): the corners of an interior window lie within WIN_GUARD - 16
// flat bytes (28 plane bytes) of the grid, and the three-word read that fetches 8 of them reaches at most 4 bytes past
// the last one, so an interior beam reads zeros there and never enters the next plane.  pool_bytes is what the bound
// pass stages; pool_fits says whether the image and its guards fit k_sweep_bound's shared memory (its static shared
// memory is below k_sweep_window's, so the window kernel's budget covers it).  Without the 4x4 image there is no
// pruning, without the 7x7 one no group pass.
constexpr int POOL_PAD = 32;
inline int pool_lead(int width_step, int K = 4) { return (K == 4 ? 4 : 8) * width_step; }
inline int pool_plane(const b2s_grid_info &g, int K = 4) { return ((pool_lead(g.width_step, K) + g.data_size) / 4 + POOL_PAD + 15) & ~15; }
inline int pool_bytes(const b2s_grid_info &g, int K = 4) { return 4 * pool_plane(g, K); }
inline int pool7_bytes(const b2s_grid_info &g) { return pool_bytes(g, 7); }
inline bool pool_fits(const b2s_grid_info &g, int smem_optin, size_t win_static, int K = 4) {
  return (long long)pool_bytes(g, K) + 2 * WIN_GUARD <= (long long)smem_optin - (long long)win_static - 512;
}
// the K x K image's layout, as the handle keeps it from create on (pitch: the per-match stride of its buffer)
struct PoolLayout { int lead, plane, bytes; size_t pitch; bool fits; };
inline PoolLayout pool_layout(const b2s_grid_info &g, int K, int smem_optin, size_t win_static) {
  const int bytes = pool_bytes(g, K);
  return {pool_lead(g.width_step, K), pool_plane(g, K), bytes, ((size_t)bytes + 127) & ~(size_t)127,
          pool_fits(g, smem_optin, win_static, K)};
}
// the byte of the staged pooled image that holds P[f]
__host__ __device__ __forceinline__ int pool_index(int f, int lead, int plane) {
  const int j = f + lead;
  return (j & 3) * plane + (j >> 2);
}
// doubles per match of the per-cell maxima plane (m_pSearchSpaceProbs), rows padded to 8
inline size_t probs_len(int search_side) { return (size_t)((search_side + 7) & ~7) * search_side; }

// ScanMatcher::Create (Mapper.cpp:126-172) + CorrelationGrid ctor (Mapper.h:920-1027) + Grid::Resize (Karto.h:4438)
inline b2s_grid_info grid_layout(const b2s_matcher_params &p) {
  b2s_grid_info g;
  uint32_t side = cast_u32(kround(p.search_size / p.resolution) + 1);
  uint32_t margin = cast_u32(ceil(p.range_threshold / p.resolution));
  int32_t grid_size = (int32_t)(side + 2 * margin);
  int32_t half_kernel = cast_i32(kround(2.0 * p.smear_deviation / p.resolution));
  uint32_t border = (uint32_t)(half_kernel + 1);
  g.width = grid_size + 2 * (int32_t)border;
  g.height = grid_size + 2 * (int32_t)border;
  g.width_step = (int32_t)(((size_t)g.width + 7) & ~(size_t)7);
  g.data_size = g.width_step * g.height;
  g.roi_x = g.roi_y = (int32_t)border;
  g.roi_w = g.roi_h = grid_size;
  g.kernel_size = 2 * half_kernel + 1;
  g.search_side = (int32_t)side;
  return g;
}

struct SweepPlan {
  b2s_status status = B2S_OK;  // not B2S_OK: the search is refused for the reason in `error`, before any launch
  const char *error = nullptr;
  int nx = 0, ny = 0, na = 0;  // candidate lattice; na = the angles THIS call sweeps (a subset when the sweep is split)
  int stride = 0;              // candidate stride in grid cells: 1, 2, or 0 (neither: generic kernel only)
  bool use_window = false;     // k_sweep_window (+ k_offsets_sorted); otherwise k_sweep_generic
  bool need_plain_lut = false; // the generic sweep and the angular covariance read the plain [nA][N] table
  // window kernel: tiles of 32 candidate rows; a grid larger than shared memory is swept in nbands row bands of
  // band_rows origin rows + halo_rows rows each, the first neg_bands of them for origins before row 0
  int copy_bytes = 0, tiles_x = 0, tiles_y = 0, rows_total = 0, halo_rows = 0;
  int band_rows = 0, nbands = 1, band_bytes = 0, neg_bands = 0;
  size_t win_smem = 0;  // dynamic shared memory of the sweep: band image + guards
  bool gen = false;     // k_sweep_window<., true>: the lanes' row starts are not two per bank
  int ctas = 0;         // persistent sweep CTAs
  // list stage (k_offsets_sorted)
  bool skip_empty = false;  // drop empty windows through the block summed-area table
  size_t osm = 0;           // its dynamic shared memory
  // angle pruning (run_correlate): a bound pass over the max-pooled grid, an exact probe of the PRUNE_PROBE angles with
  // the largest bounds, then an exact sweep of only the angles whose bound reaches the probe's best response - 0.1
  bool prune = false;
  // k_sweep_bound places every beam itself: it stages the scan-local points (and, with skip_empty, the summed-area
  // table) in shared memory after the pooled image when they fit there, and reads them through L1 otherwise
  bool bound_stage = false;
  size_t bound_smem = 0;  // dynamic shared memory of k_sweep_bound: pooled image + guards (+ points + SAT when staged)
  // the group pass (k_sweep_bound_group over the 7x7 image) runs first, and k_sweep_bound bounds single angles only
  // where a group's bound can matter; without it every group counts as unbounded and k_sweep_bound bounds every angle
  bool group = false;
  bool group_stage = false;  // the group pass stages the scan-local points after its image
  size_t group_smem = 0;     // its dynamic shared memory: 7x7 image + guards (+ points when staged)
  // the accumulators of split_chunks, up to 2 * warps - 1 of them (a round of more units is not split): the bound's
  // per-unit rows of block sums, BOUND_ROW_BYTES each after bound_smem / group_smem (0: every unit is one item), and
  // the listed sweeps' ny x nx planes after the grid image
  int bound_rows = 0, group_rows = 0;
  int acc_slots = 0;
  size_t listed_smem = 0;  // win_smem + the planes
};

// shared memory k_sweep_bound stages after its pooled image (bound_stage): n scan-local points and the SAT when used
inline size_t bound_stage_bytes(int n, bool skip_empty, int sbx, int sby) {
  return (size_t)n * 2 * sizeof(double) + (skip_empty ? sizeof(uint16_t) * sat_stride(sbx, sby) : 0);
}

// p, g: the handle's parameters and grid; n: beams; k_first / na_override: the angle subset of a split sweep
// (na_override < 0: every angle); force_kernel: b2s_matcher_set_kernel; sat_valid / grid_high_bytes / sbx / sby: the
// state of the grids; num_sms, smem_optin: the device's; win_static: the sweep kernel's static shared memory.
inline SweepPlan plan_sweep(const b2s_matcher_params &p, const b2s_grid_info &g, const b2s_search &s, int n, int batch,
                            int k_first, int na_override, int force_kernel, bool sat_valid, bool grid_high_bytes,
                            int sbx, int sby, int num_sms, int smem_optin, size_t win_static) {
  SweepPlan pl;
  auto refuse = [&pl](b2s_status st, const char *why) {
    pl.status = st;
    pl.error = why;
    return pl;
  };
  if (s.angle_res == 0.0 || s.res_x == 0.0 || s.res_y == 0.0)
    return refuse(B2S_ERR_BAD_PARAMS, "search resolutions must be non-zero");  // assert at Mapper.cpp:319
  pl.nx = n_steps(s.offset_x, s.res_x);
  pl.ny = n_steps(s.offset_y, s.res_y);
  const int na_full = n_steps(s.angle_offset, s.angle_res);
  pl.na = na_override >= 0 ? na_override : na_full;
  if (k_first < 0 || k_first + pl.na > na_full) return refuse(B2S_ERR_BAD_PARAMS, "angle subset outside the search");
  if (pl.nx <= 0 || pl.ny <= 0 || na_full <= 0 || (long long)pl.nx * pl.ny * std::max(pl.na, 1) > (1ll << 28))
    return refuse(B2S_ERR_TOO_LARGE, "search volume too large");

  // The window kernel needs a stride-1 or stride-2 lattice and a band of the grid in shared memory: the whole grid when
  // it fits (nbands = 1), otherwise nbands row bands.
  pl.copy_bytes = (g.data_size + 15) & ~15;
  // candidate stride in grid cells: 1 (search resolution == grid resolution) or 2 (the coarse stage of MatchScan,
  // Mapper.cpp:233-234); anything else goes to the generic kernel
  const double gres = 1.0 / (1.0 / p.resolution);
  auto stride_of = [&](double r) { return (r == gres || r == p.resolution) ? 1 : ((r == 2 * gres || r == 2 * p.resolution) ? 2 : 0); };
  pl.stride = (stride_of(s.res_x) == stride_of(s.res_y)) ? stride_of(s.res_x) : 0;
  const int stride1 = std::max(pl.stride, 1);
  const int cpt = pl.stride == 2 ? 16 : 32;  // candidates per 32-byte tile row
  pl.tiles_x = (pl.nx + cpt - 1) / cpt;
  pl.tiles_y = (pl.ny + 31) / 32;
  pl.rows_total = pl.tiles_y * 32;
  pl.halo_rows = stride1 * 31 + 2;  // rows below the first row of a 32-row candidate tile that a lane may touch
  const long long smem_limit = (long long)smem_optin - (long long)win_static - 512;
  pl.band_rows = std::max(g.height, 1);
  pl.band_bytes = pl.copy_bytes;
  bool bands_ok = true;
  if ((long long)pl.copy_bytes + 2 * WIN_GUARD > smem_limit) {
    const long long rows_fit = (smem_limit - 2 * WIN_GUARD) / g.width_step;
    pl.band_rows = (int)((rows_fit - pl.halo_rows) & ~1LL);  // even: band starts stay 16-byte aligned (width_step % 8 == 0)
    if (pl.band_rows < 8) {
      bands_ok = false;
    } else {
      // origins up to (window rows) below the grid still reach it from their upper row tiles: bands of their own
      pl.neg_bands = pl.tiles_y > 1 ? (stride1 * (pl.rows_total - 1) + 1 + pl.band_rows - 1) / pl.band_rows : 0;
      pl.nbands = (g.height + pl.band_rows - 1) / pl.band_rows + pl.neg_bands;
      pl.band_bytes = (int)((long long)(pl.band_rows + pl.halo_rows) * g.width_step);
      if (pl.nbands > WIN_MAX_BANDS) bands_ok = false;
    }
  }
  pl.win_smem = (size_t)((pl.band_bytes + 15) & ~15) + 2 * WIN_GUARD;
  const bool win_fits = bands_ok && pl.stride != 0 && (g.width_step % 8) == 0 && n > 0 &&
                        (size_t)n * OFF_SMEM_PER_BEAM + 64 <= LIST_SMEM_MAX && !grid_high_bytes;
  if (force_kernel >= 2 && !win_fits)
    return refuse(B2S_ERR_TOO_LARGE, "window kernel forced but not applicable to this lattice / grid / beam count");
  pl.use_window = force_kernel >= 2 || (win_fits && force_kernel != 1);
  pl.need_plain_lut = !pl.use_window || s.fine;
  if (s.fine && sizeof(double) * (size_t)pl.na > 48 * 1024)
    return refuse(B2S_ERR_TOO_LARGE, "too many angles for the angular-covariance kernel");

  const size_t beams_bytes = ((size_t)n * OFF_SMEM_PER_BEAM + 15) & ~(size_t)15;
  const size_t sat_bytes = sizeof(uint16_t) * sat_stride(sbx, sby);
  pl.skip_empty = sat_valid && force_kernel != 3 && beams_bytes + sat_bytes + 64 <= LIST_SMEM_MAX;
  pl.osm = beams_bytes + (pl.skip_empty ? sat_bytes : 0) + 64;
  pl.ctas = (int)std::min<long long>((long long)batch * pl.nbands * (pl.nbands > 1 ? pl.tiles_y : 1), num_sms);
  // the GEN = false instantiation assumes exactly two lanes per row-start bank (see win_load)
  const int bank_step = ((g.width_step >> 2) * stride1) & 31;
  pl.gen = (bank_step & 3) != 2;
  // Pruning needs the whole grid and the whole pooled image in shared memory, one 32 x 32 stride-1 candidate tile (the
  // bound's 8 x 8 blocks of 4 x 4 candidates), and the whole angle range of a search: an angle subset of a split sweep
  // cannot know the global best.  Selector 3 sweeps every beam and every angle.
  const PoolLayout pool = pool_layout(g, 4, smem_optin, win_static), pool7 = pool_layout(g, 7, smem_optin, win_static);
  pl.bound_smem = (size_t)pool.bytes + 2 * WIN_GUARD;
  pl.prune = pl.use_window && pl.nbands == 1 && pl.stride == 1 && pl.tiles_x == 1 && pl.tiles_y == 1 &&
             na_override < 0 && force_kernel != 3 && pl.na >= PRUNE_MIN_ANGLES && pl.na <= PRUNE_MAX_ANGLES && pool.fits;
  pl.group = pl.prune && pool7.fits;
  pl.group_smem = (size_t)pool7.bytes + 2 * WIN_GUARD;
  // a pass that runs stages `staged` bytes after its image of `smem` bytes when both fit
  auto stage = [&](bool runs, size_t &smem, size_t staged) {
    const bool fits = runs && (long long)(smem + staged) <= smem_limit;
    if (fits) smem += staged;
    return fits;
  };
  pl.bound_stage = stage(pl.prune, pl.bound_smem, bound_stage_bytes(n, pl.skip_empty, sbx, sby));
  pl.group_stage = stage(pl.group, pl.group_smem, bound_stage_bytes(n, false, sbx, sby));
  if (!pl.group) pl.group_smem = 0;
  // the accumulators of `unit` bytes that fit after `used` bytes
  auto accumulators = [&](size_t used, long long unit) {
    const long long room = std::max(smem_limit - (long long)used, 0LL);
    return (int)std::min<long long>(2 * (WIN_THREADS / 32) - 1, room / unit);
  };
  if (pl.prune) pl.bound_rows = accumulators(pl.bound_smem, BOUND_ROW_BYTES);
  if (pl.group) pl.group_rows = accumulators(pl.group_smem, BOUND_ROW_BYTES);
  if (pl.prune) {
    const long long plane = 4LL * pl.nx * pl.ny;
    pl.acc_slots = accumulators(pl.win_smem, plane);
    pl.listed_smem = pl.win_smem + (size_t)(pl.acc_slots * plane);
  }
  return pl;
}

}  // namespace b2s
