/*
 * b200slam.h — the C ABI of the H100-native 2-D laser SLAM front-end hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8(b)).  The reference
 * (xiangli0608/Creating-2D-laser-slam-from-scratch) has no C ABI; its seams are C++ class
 * methods called in-process.  Every entry point below names the reference method it stands in
 * for (file:line relative to the reference checkout).  A reference-side façade with the reference's own
 * signatures is in include/b200slam/karto_facade.hpp; INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types; all arrays are caller-owned HOST memory
 *     unless the name says `_device`.
 *   - every function returns a b2s_status (0 = OK); exceptions of the reference map to codes.
 *   - a handle is single-threaded like the reference's ScanMatcher (Mapper.h:1273-1278 shares
 *     m_pCorrelationGrid / m_pGridLookup); DISTINCT handles may be used concurrently
 *     (one CUDA stream each).
 *   - "batch" = B independent scan-matches, each with its OWN correlation grid (SURVEY.md §8(e)(i)).
 *   - poses are (x, y, heading) doubles; covariances are row-major 3x3 doubles.
 *   - the product path is CUDA only: if no device is usable every compute entry point returns
 *     B2S_ERR_NO_DEVICE.  There is no CPU fallback.
 */
#ifndef B200SLAM_H
#define B200SLAM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_ABI_VERSION 1

typedef enum b2s_status {
  B2S_OK = 0,
  B2S_ERR_BAD_PARAMS = 1,   /* ScanMatcher::Create -> NULL (Mapper.cpp:130-145); smear out of range (Mapper.h:1045-1053) */
  B2S_ERR_OUT_OF_RANGE = 2, /* karto::Exception "Index out of range" (Karto.h:4492-4498) */
  B2S_ERR_NO_BEST_POSE = 3, /* std::runtime_error "Unable to find best position" (Mapper.cpp:486) */
  B2S_ERR_CUDA = 4,         /* a CUDA runtime call failed; see b2s_last_error() */
  B2S_ERR_NO_DEVICE = 5,    /* no CUDA device: the product path never falls back to the CPU */
  B2S_ERR_BAD_STATE = 6,    /* call order violated (e.g. correlate before scans are set) */
  B2S_ERR_TOO_LARGE = 7     /* batch / beam count / window exceeds what the handle was created for */
} b2s_status;

/* ScanMatcher::Create arguments (Mapper.cpp:126-127) + the 8 tuning values the matcher reads from its
 * Mapper through friend access (Mapper.cpp:206,238-239,250,256,279-280,405-411).  Values are the ones
 * STORED in the Mapper: setParamDistanceVariancePenalty/AngleVariancePenalty square their argument
 * (Mapper.cpp:1919-1927) — do that before filling this struct.  Defaults: Mapper.cpp:1569-1652. */
typedef struct b2s_matcher_params {
  double search_size;                /* CorrelationSearchSpaceDimension, m */
  double resolution;                 /* CorrelationSearchSpaceResolution, m/cell */
  double smear_deviation;            /* CorrelationSearchSpaceSmearDeviation, m */
  double range_threshold;            /* LaserRangeFinder range threshold, m */
  double distance_variance_penalty;  /* default 0.3^2 */
  double angle_variance_penalty;     /* default (20 deg)^2 */
  double fine_search_angle_offset;   /* default 0.2 deg */
  double coarse_search_angle_offset; /* default 20 deg */
  double coarse_angle_resolution;    /* default 2 deg */
  double minimum_angle_penalty;      /* default 0.9 */
  double minimum_distance_penalty;   /* default 0.5 */
  int32_t use_response_expansion;    /* default 0 */
  int32_t reserved;
} b2s_matcher_params;

/* The part of karto::LaserRangeFinder (Karto.h:3700-4184) the hot path reads. */
typedef struct b2s_laser {
  int32_t n_readings; /* LaserRangeFinder::GetNumberOfRangeReadings (1081 for Hokuyo_UTM_30LX; a Custom
                         sensor yields round((max-min)/res) WITHOUT +1, Karto.h:4158-4160) */
  int32_t reserved;
  double min_angle;          /* rad */
  double angular_resolution; /* rad */
  double min_range;          /* m */
  double max_range;          /* m */
  double range_threshold;    /* m */
  double offset_pose[3];     /* sensor pose in the robot frame (Sensor::GetOffsetPose) */
} b2s_laser;

/* CorrelationGrid geometry (Mapper.h:900-1118, Karto.h:4381-4767). */
typedef struct b2s_grid_info {
  int32_t width, height; /* allocation incl. smear border */
  int32_t width_step;    /* AlignValue(width, 8) (Karto.h:4442) */
  int32_t data_size;     /* width_step * height bytes */
  int32_t roi_x, roi_y, roi_w, roi_h;
  int32_t kernel_size;   /* smear kernel side, 2*round(2*sigma/res)+1 */
  int32_t search_side;   /* m_pSearchSpaceProbs side = round(search_size/res)+1 */
} b2s_grid_info;

/* CorrelateScan arguments (Mapper.cpp:309-317), shared by every match of a batch. */
typedef struct b2s_search {
  double offset_x, offset_y;   /* rSearchSpaceOffset */
  double res_x, res_y;         /* rSearchSpaceResolution */
  double angle_offset;         /* searchAngleOffset */
  double angle_res;            /* searchAngleResolution */
  int32_t do_penalize;
  int32_t fine;                /* doingFineMatch */
} b2s_search;

typedef struct b2s_match_result {
  double response;   /* return value of CorrelateScan / MatchScan, clamped to <= 1 */
  double pose[3];    /* rMean */
  double cov[9];     /* rCovariance, row-major */
  int32_t status;    /* per-match b2s_status (B2S_ERR_NO_BEST_POSE ...) */
  int32_t tie_count; /* averagePoseCount (Mapper.cpp:459-471) */
} b2s_match_result;

typedef struct b2s_matcher b2s_matcher; /* opaque: replaces karto::ScanMatcher* */

/* ---------------------------------------------------------------- library */
int b2s_abi_version(void);
const char *b2s_last_error(void);              /* thread-local text of the last failure */
int b2s_device_count(void);                    /* 0 when no usable CUDA device */

/* ---------------------------------------------------------------- K1: Karto correlative scan matcher
 * Host arrays are caller-owned.  Uploads are enqueued on the handle's stream: out of pageable memory the CUDA runtime
 * stages them before the call returns; out of PINNED memory they are asynchronous, so such buffers must stay unchanged
 * until the next call that waits for the stream (correlate_scan, match_scan, _end, sync). */

/* ScanMatcher::Create (Mapper.cpp:126-172).  `max_batch` matches share one handle, each with up to
 * `max_base_scans` base scans; `max_batch` may be any count >= 1 whose buffers fit in device memory (65 535 is not a
 * limit).  Buffers that depend on the search volume grow on demand.  `cuda_stream` may be NULL
 * (the handle then creates its own non-blocking stream) or a cudaStream_t owned by the caller. */
b2s_status b2s_matcher_create(const b2s_matcher_params *params, const b2s_laser *laser, int device,
                              int max_batch, int max_base_scans, void *cuda_stream, b2s_matcher **out);
void b2s_matcher_destroy(b2s_matcher *m);      /* ScanMatcher::~ScanMatcher (Mapper.cpp:119-124) */
b2s_status b2s_matcher_grid_info(const b2s_matcher *m, b2s_grid_info *out);

/* The scans being matched: B x (ranges[n_readings], robot pose).  Replaces building B
 * LocalizedRangeScan objects + SetOdometricPose/SetCorrectedPose (karto_slam.cc:437-440).
 * Point readings are derived on the device as LocalizedRangeScan::Update does (Karto.h:5362-5428). */
b2s_status b2s_matcher_set_scans(b2s_matcher *m, int batch, const double *ranges, const double *poses);

/* MatchScan steps 1-4 + AddScans (Mapper.cpp:195-225, 699-811; Mapper.h:971-1005): centre grid b on scan
 * b's sensor pose and rasterise + smear its `n_base` base scans.  base_ranges: [batch][n_base][n_readings],
 * base_poses: [batch][n_base][3].  Any beam count is accepted: scans too long for the parallel kernel's shared memory
 * (more than about 9 300 beams on an H100) are rasterised by the sequential kernel, with the same grid bytes. */
b2s_status b2s_matcher_add_scans(b2s_matcher *m, int n_base, const double *base_ranges, const double *base_poses);

/* Scan pool: readings that serve as base scans of many matches (a mapper's running window, near chains, loop-closure
 * candidate chains) are uploaded once (_pool_append returns the row) and referenced by row afterwards;
 * _add_scans_pool is b2s_matcher_add_scans with pool rows ([batch][n_base], host) in place of base_ranges. */
b2s_status b2s_matcher_pool_append(b2s_matcher *m, const double *ranges, int32_t *out_row);
int32_t b2s_matcher_pool_count(const b2s_matcher *m);
b2s_status b2s_matcher_add_scans_pool(b2s_matcher *m, int n_base, const int32_t *pool_rows, const double *base_poses);

/* Alternative to add_scans for callers that keep grids themselves: upload ready-made correlation grids
 * ([batch][data_size] bytes) and their world offsets ([batch][2], CoordinateConverter::SetOffset). */
b2s_status b2s_matcher_set_grids(b2s_matcher *m, const uint8_t *grids, const double *offsets);

/* ScanMatcher::CorrelateScan (Mapper.cpp:309-523) for every match of the batch; centers: [batch][3].
 * For fine=1 results[b].cov is IN/OUT exactly like rCovariance (only cov[8] is overwritten, Mapper.cpp:648,691). */
b2s_status b2s_matcher_correlate_scan(b2s_matcher *m, const double *centers, const b2s_search *search,
                                      b2s_match_result *results);

/* The same call split in two so that a caller can pipeline batches on two handles (one batch's uploads, rasterisation and
 * lookup lists overlap the other batch's sweep): _begin enqueues everything incl. the result read-back on the handle's
 * stream and returns; _end waits and hands the results out.  cov_in is only read for fine = 1 (may be NULL otherwise).
 * Host buffers handed to set_scans / add_scans / _begin must stay unchanged until _end returns when they are pinned
 * (uploads out of pinned memory are asynchronous). */
b2s_status b2s_matcher_correlate_scan_begin(b2s_matcher *m, const double *centers, const b2s_search *search,
                                            const b2s_match_result *cov_in);
b2s_status b2s_matcher_correlate_scan_end(b2s_matcher *m, b2s_match_result *results);

/* ScanMatcher::MatchScan (Mapper.cpp:184-291): coarse sweep (+ optional response expansion) + fine sweep.
 * Requires set_scans + add_scans (or set_grids). */
b2s_status b2s_matcher_match_scan(b2s_matcher *m, int do_penalize, int do_refine, b2s_match_result *results);

/* One-call host-buffer form (what a reference node's MatchScan call costs end to end):
 * set_scans + add_scans + match_scan. */
b2s_status b2s_matcher_match_scan_host(b2s_matcher *m, int batch, const double *ranges, const double *poses,
                                       int n_base, const double *base_ranges, const double *base_poses,
                                       int do_penalize, int do_refine, b2s_match_result *results);

/* A coarse CorrelateScan whose ANGLES are split over several GPUs (SURVEY.md §8(e)(ii)): every rank holds the same
 * scans + grids and sweeps angle indices [k_first, k_first + k_count).  Between the three phases the caller
 * all-reduces the small host arrays (NCCL via torch.distributed in creating-..._b200/parallel.py):
 *   begin : best[batch] (MAX), probs[batch][probs_len] per-cell maxima plane (MAX), status[batch] (MAX);
 *           probs_len = AlignValue(search_side, 8) * search_side
 *   ties  : global best in; tie_sums[batch][5] = {sum x, sum y, sum cos, sum sin, count} out (SUM)
 *   finish: global best / tie sums / plane in; results as b2s_matcher_correlate_scan (positional covariance incl.) */
b2s_status b2s_matcher_correlate_split_begin(b2s_matcher *m, const double *centers, const b2s_search *search, int k_first,
                                             int k_count, double *best, double *probs, int32_t *status);
b2s_status b2s_matcher_correlate_split_ties(b2s_matcher *m, const double *global_best, double *tie_sums);
b2s_status b2s_matcher_correlate_split_finish(b2s_matcher *m, const double *global_best, const double *tie_sums,
                                              const double *probs, b2s_match_result *results);

/* Inspection (parity tests; also ScanMatcher::GetCorrelationGrid, Mapper.h:1192). */
b2s_status b2s_matcher_get_grid(b2s_matcher *m, int b, uint8_t *out_bytes, double out_offset[2]);
b2s_status b2s_matcher_get_point_readings(b2s_matcher *m, int b, double *out_xy /* [n_readings][2] */);
/* GridIndexLookup::ComputeOffsets (Karto.h:6409-6501): out[n_angles][n_readings]; INT32_MAX = INVALID_SCAN */
b2s_status b2s_matcher_compute_offsets(b2s_matcher *m, int b, double angle_center, double angle_offset,
                                       double angle_res, int32_t *out, int32_t *out_n_angles);
/* integer numerators of GetResponse (Mapper.cpp:819-856) of the LAST correlate_scan sweep for match b,
 * in the reference's loop order out[nY][nX][nAngles] (Mapper.cpp:373-424). */
/* The angle-split sweep with the collectives INSIDE the library: nccl_comm is the caller's ncclComm_t (the library
 * dlopens libnccl.so.2 and calls ncclAllReduce on the handle's stream; no host staging, no Python).  Every rank calls
 * it with the same scans / grids / centres and its own rank; results are those of b2s_matcher_correlate_scan on
 * every rank.  Collectives: best response MAX (B doubles), per-cell plane MAX (B x probs_len doubles), status MAX,
 * tie sums SUM (5B doubles). */
b2s_status b2s_matcher_correlate_scan_split(b2s_matcher *m, void *nccl_comm, int rank, int world, const double *centers,
                                            const b2s_search *search, b2s_match_result *results);
/* ms of its last call: all-reduce(best), all-reduce(plane + status), all-reduce(tie sums), sweep end -> results */
b2s_status b2s_matcher_last_split_timing(b2s_matcher *m, double out[4]);
b2s_status b2s_matcher_get_response_sums(b2s_matcher *m, int b, int32_t *out, int32_t dims[3]);

/* Device time (ms, CUDA events on the handle's stream) of the stages of the LAST correlate_scan call:
 * out[0] = offsets/LUT, out[1] = response sweep, out[2] = reduce (max / tie-average / covariance),
 * out[3] = number of sweep kernel launches. */
b2s_status b2s_matcher_last_timing(b2s_matcher *m, double out[4]);
/* Statistics of the LAST correlate_scan call: out[0] = fraction of (beam, angle) windows the window kernel dropped
 * because every cell of the nY x nX window lies in empty 4x4 blocks of the grid (they add 0 to every candidate, so
 * results are unchanged); out[1] = sweep path (1 generic, 2 window); out[2] = candidates per match; out[3] = beams. */
b2s_status b2s_matcher_last_stats(b2s_matcher *m, double out[4]);
/* Fraction of the (match, angle) pairs of the LAST correlate_scan call that the window kernel never swept because an
 * upper bound of all their responses lies below best - 0.1 (results unchanged; 0 when the search was not pruned). */
b2s_status b2s_matcher_last_pruned_frac(b2s_matcher *m, double *out);
/* Angle-pruning state of the LAST sweep (tests): the last correlate_scan call, or the last stage of the last
 * match_scan / match_scan_host / split call.  ubr [B][nA] (NaN where the angle was not bounded one by one),
 * gub [B][ceil(nA / 4)], swept [B][nA] (1 = swept exactly), cut [B].  dims = {B, nA} the caller's arrays are sized
 * for; on return it holds the last sweep's, and a call with every array null only reports them.  B2S_ERR_BAD_PARAMS
 * (nothing written to the arrays) when they differ; B2S_ERR_BAD_STATE when that sweep was not pruned,
 * b2s_matcher_get_response_sums has re-swept it since, or set_scans / add_scans / set_grids replaced its inputs.
 * Null arrays are skipped.
 * cut[b] = L - 0.1 - 1e-9, L the best exact response of the probed angles; when L - 0.1 <= 1e-6 every angle is swept
 * and cut[b] still holds that value.  A match the generic kernel swept (an irregular candidate lattice, or no result)
 * is not bounded: its ubr row and cut are NaN, its swept row all 1, and its gub row holds whatever the group pass
 * left there (nothing it was compared with).  Without the group pass (SweepPlan::group) every gub is 0x7f7f... as
 * a double (about 1.4e306): every group is bounded one angle at a time. */
b2s_status b2s_matcher_last_prune_state(b2s_matcher *m, int32_t dims[2], double *ubr, double *gub, uint8_t *swept,
                                        double *cut);
b2s_status b2s_matcher_sync(b2s_matcher *m);
/* 0 = automatic, 1 = force the generic global-memory gather kernel, 2 = force the shared-memory window kernel,
 * 3 = window kernel over every beam and every angle (no empty-window dropping, no angle pruning) */
b2s_status b2s_matcher_set_kernel(b2s_matcher *m, int which);

/* ---------------------------------------------------------------- lesson6 front end: karto::Mapper / MapperGraph
 * The host driver that feeds K1 (SURVEY.md §8(f).1): key-frame gate, running-scan window, sequential MatchScan,
 * pose-graph vertices / edges, near-chain links and loop-closure candidates (Mapper.cpp:883-1414, 1999-2125;
 * Mapper.h:1288-1404).  Every MatchScan runs on the device; independent matches of one Process call (all near
 * chains of LinkNearChains, all candidate chains of TryCloseLoop up to the first accepted closure) go out as ONE
 * batch.  Several sensors (robots) may feed one mapper: b2s_mapper_process_sensor (MapperSensorManager semantics, the
 * first-scan linking of Mapper.cpp:920-952 included). */

/* Values as the Mapper STORES them (Mapper.cpp:1448-1653); the setParam* squaring of distance_variance_penalty,
 * angle_variance_penalty and loop_match_maximum_variance_coarse (Mapper.cpp:1871-1874,1919-1927) is the caller's job. */
typedef struct b2s_mapper_params {
  int32_t use_scan_matching;                 /* true */
  int32_t use_scan_barycenter;               /* true */
  double minimum_time_interval;              /* 3600 s */
  double minimum_travel_distance;            /* 0.2 m */
  double minimum_travel_heading;             /* 10 deg in rad */
  int32_t scan_buffer_size;                  /* 70 */
  int32_t do_loop_closing;                   /* true */
  double scan_buffer_maximum_scan_distance;  /* 20 m */
  double link_match_minimum_response_fine;   /* 0.8 */
  double link_scan_maximum_distance;         /* 10 m */
  double loop_search_maximum_distance;       /* 4 m */
  int32_t loop_match_minimum_chain_size;     /* 10 */
  int32_t reserved;
  double loop_match_maximum_variance_coarse; /* 0.4^2 */
  double loop_match_minimum_response_coarse; /* 0.8 */
  double loop_match_minimum_response_fine;   /* 0.8 */
  b2s_matcher_params sequential;             /* CorrelationSearchSpace* 0.3 / 0.01 / 0.03 + the shared tuning values */
  b2s_matcher_params loop;                   /* LoopSearchSpace* 8.0 / 0.05 / 0.03 + the same tuning values */
} b2s_mapper_params;

/* Mapper::InitializeParameters defaults (Mapper.cpp:1448-1653); range_threshold of both matchers = the laser's */
void b2s_mapper_default_params(b2s_mapper_params *out, double range_threshold);

/* The matcher plug-in: ScanMatcher::MatchScan (Mapper.cpp:184-291) for a batch of independent matches.
 * which = 0 the sequential matcher (Mapper::m_pSequentialScanMatcher), 1 the loop matcher
 * (MapperGraph::m_pLoopScanMatcher).  ranges [batch][N], poses [batch][3] (robot poses); the base scans of match b are
 * base_ranges/base_poses[base_first[b] .. base_first[b] + n_base[b]).  The in-tree implementation is the CUDA matcher
 * (b2s_mapper_create); the hook exists so that the graph logic can be exercised without a device. */
typedef b2s_status (*b2s_match_scan_fn)(void *user, int which, int batch, const double *ranges, const double *poses,
                                        const int32_t *base_first, const int32_t *n_base, const double *base_ranges,
                                        const double *base_poses, int do_penalize, int do_refine,
                                        b2s_match_result *results);

/* karto::ScanSolver (Mapper.h:825-891) as a C vtable — the reference's own back-end plug-in interface. */
typedef struct b2s_scan_solver {
  void *user;
  void (*add_node)(void *user, int32_t unique_id, const double corrected_pose[3]);          /* AddNode */
  void (*add_constraint)(void *user, int32_t source_id, int32_t target_id, const double pose_difference[3],
                         const double covariance[9]);                                       /* AddConstraint(LinkInfo) */
  int32_t (*compute)(void *user, int32_t capacity, int32_t *ids, double *poses /* [capacity][3] */);
                                                                                             /* Compute + GetCorrections */
  void (*clear)(void *user);                                                                /* Clear */
} b2s_scan_solver;

typedef struct b2s_mapper b2s_mapper; /* opaque: replaces karto::Mapper (+ MapperGraph, MapperSensorManager) */

b2s_status b2s_mapper_create(const b2s_mapper_params *params, const b2s_laser *laser, int device, b2s_mapper **out);
b2s_status b2s_mapper_create_with_matcher(const b2s_mapper_params *params, const b2s_laser *laser,
                                          b2s_match_scan_fn match, void *user, b2s_mapper **out);
void b2s_mapper_destroy(b2s_mapper *m);
/* Mapper::SetScanSolver (Mapper.cpp:2220); NULL = no back end (poses are never corrected, as with use_back_end false) */
b2s_status b2s_mapper_set_scan_solver(b2s_mapper *m, const b2s_scan_solver *solver);
/* Mapper::Process(LocalizedRangeScan*) (Mapper.cpp:1999-2079): ranges[n_readings], odometric robot pose, time stamp (s).
 * out_processed = the kt_bool it returns (false: rejected by HasMovedEnough); out_corrected_pose = GetCorrectedPose().
 * A non-OK status returned after the scan entered the graph (edge building / loop closing failed: CUDA error,
 * B2S_ERR_NO_BEST_POSE, or B2S_ERR_BAD_STATE where the reference's Matrix3::Inverse asserts) leaves the mapper where
 * the reference process would have aborted: the handle is marked failed, later calls return B2S_ERR_BAD_STATE, and it
 * must be destroyed. */
b2s_status b2s_mapper_process(b2s_mapper *m, const double *ranges, const double odometric_pose[3], double time,
                              int32_t *out_processed, double out_corrected_pose[3]);
/* The same for a scan of the NAMED sensor (LocalizedRangeScan::GetSensorName; karto_slam.cc passes the laser frame id).
 * MapperSensorManager semantics (Mapper.h:1412-1577, Mapper.cpp:45-100): a sensor is registered by its first scan; each
 * sensor has its own scan list (state ids), running window and last scan, unique ids count over all sensors; a sensor's
 * first scan is matched against ALL scans of every other sensor (name order = Name::operator<, Karto.h:484) and linked
 * to that sensor's first scan (Mapper.cpp:920-952); near chains follow the near scan's own sensor and loop closures are
 * searched against every sensor's scans in name order (Mapper.cpp:2063-2070).  All sensors share the handle's b2s_laser
 * (same LaserRangeFinder parameters on every robot).  b2s_mapper_process is this call with the name "laser". */
b2s_status b2s_mapper_process_sensor(b2s_mapper *m, const char *sensor_name, const double *ranges,
                                     const double odometric_pose[3], double time, int32_t *out_processed,
                                     double out_corrected_pose[3]);
int32_t b2s_mapper_sensor_count(const b2s_mapper *m);
/* per processed scan (unique-id order): the rank of its sensor in name order, [count] */
b2s_status b2s_mapper_get_scan_sensors(const b2s_mapper *m, int32_t *out);
int32_t b2s_mapper_scan_count(const b2s_mapper *m);   /* GetAllProcessedScans().size() */
/* corrected poses of every processed scan in unique-id order, [count][3] (they move when a loop closes and a solver is
 * set) */
b2s_status b2s_mapper_get_poses(const b2s_mapper *m, double *out);
int32_t b2s_mapper_edge_count(const b2s_mapper *m);
/* graph edges in creation order: ids [count][2] (source, target), LinkInfo pose difference [count][3] and covariance
 * [count][9] (Mapper.h:108-175) */
b2s_status b2s_mapper_get_edges(const b2s_mapper *m, int32_t *ids, double *pose_difference, double *covariance);
/* out[0] = MatchScan calls so far, out[1] = device batches they were sent in, out[2] = loop-closure candidate chains
 * examined, out[3] = loops closed, out[4] = running-scan window size of the sensor processed last */
b2s_status b2s_mapper_stats(const b2s_mapper *m, double out[5]);

/* ---------------------------------------------------------------- back end: a ScanSolver for the mapper (host only)
 * SURVEY.md §8(f).3: the reference's back ends (sparse bundle adjustment / g2o / Ceres / GTSAM, lesson6/src/<name>_solver)
 * need Eigen + SuiteSparse and stay on the CPU in every BASELINE config.  This is a small dependency-free 2-D pose-graph
 * optimiser with the same role: nodes = scan poses, constraints = LinkInfo pose differences weighted by the inverse
 * covariance (lesson6/src/spa_solver/spa_solver.cc:65-93), Levenberg-Marquardt outer loop, block-Jacobi preconditioned
 * conjugate gradients inside, first node fixed.  It is NOT a restatement of sba::SysSPA2d (parity unpinned: that
 * library is not under the reference checkout); tests plug the SAME solver into the reference Mapper and into ours. */
typedef struct b2s_pose_graph b2s_pose_graph;
b2s_status b2s_pose_graph_create(b2s_pose_graph **out);
void b2s_pose_graph_destroy(b2s_pose_graph *g);
/* fills `out` with callbacks bound to `g` (valid while g lives): pass it to b2s_mapper_set_scan_solver */
b2s_status b2s_pose_graph_as_scan_solver(b2s_pose_graph *g, b2s_scan_solver *out);
/* SpaSolver::Compute runs doSPA(40) (spa_solver.cc:44-63): max LM iterations (default 40), PCG iterations per step */
b2s_status b2s_pose_graph_set_iterations(b2s_pose_graph *g, int lm_iterations, int cg_iterations);
/* out[0] = nodes, out[1] = constraints, out[2] = chi^2 before the last Compute, out[3] = after, out[4] = LM steps taken */
b2s_status b2s_pose_graph_stats(const b2s_pose_graph *g, double out[5]);

/* ---------------------------------------------------------------- K2c: karto::OccupancyGrid */

typedef struct b2s_occ_grid_info {
  int32_t width, height, width_step, data_size;
  double offset[2];  /* CoordinateConverter offset = bounding-box minimum (Karto.h:5821) */
  double resolution;
  uint64_t cell_visits; /* Bresenham cells touched incl. end cells (SURVEY.md §8(d) V) */
} b2s_occ_grid_info;

typedef struct b2s_occ_grid b2s_occ_grid; /* opaque: replaces karto::OccupancyGrid* */

/* OccupancyGrid::CreateFromScans (Karto.h:5659-5673, 5804-5990): n_scans x (ranges, robot pose).
 * Returns B2S_OK with *out == NULL when n_scans == 0 (the reference returns NULL). */
b2s_status b2s_occ_grid_create_from_scans(const b2s_laser *laser, int n_scans, const double *ranges,
                                          const double *poses, double resolution, int device,
                                          void *cuda_stream, b2s_occ_grid **out);
/* Many grids at once: grid g = b2s_occ_grid_create_from_scans over its own n_scans[g] scans, ranges / poses grid-major
 * (grid 0's scans first), at resolution[g].  The readings are float32 ([sum n_scans][n_readings]), widened to double on
 * the device, so a grid equals b2s_occ_grid_create_from_scans over the same readings as doubles, bit for bit in info
 * and payload.  Every stage is one launch for all grids (per-scan boxes, per-grid unions, one read-back of the unions
 * to size the grids, one counter arena, one ray trace over every beam of every grid, one threshold + payload pass) and
 * the payloads come back in one copy.  on_grid(user, g, info, payload [height][width] int8 as b2s_occ_grid_copy_ros)
 * is called in ascending g for every grid with scans; a grid without scans has no map (CreateFromScans returns NULL)
 * and is skipped.  Pointers are valid only during the callback.  n_grids may be any count whose maps fit in device
 * memory (65 535 is not a limit).  B2S_ERR_BAD_PARAMS for NULL arrays, negative counts or a zero resolution of a grid
 * with scans. */
typedef void (*b2s_occ_grid_batch_fn)(void *user, int32_t grid, const b2s_occ_grid_info *info, const int8_t *payload);
b2s_status b2s_occ_grid_create_from_scans_batch(const b2s_laser *laser, int n_grids, const int32_t *n_scans,
                                                const float *ranges, const double *poses, const double *resolution,
                                                int device, b2s_occ_grid_batch_fn on_grid, void *user);
/* The same map built from a scan list SHARDED over several GPUs (SURVEY.md §8(e)(iii)): pass/hit counters are
 * commutative, so each rank ray-traces its shard into a grid sized by the GLOBAL bounding box and the counters are
 * summed (NCCL all-reduce, in place on the device pointers) before OccupancyGrid::Update thresholds them.
 *   1. b2s_occ_grid_scans_bbox  -> this shard's BoundingBox2 {min x, min y, max x, max y} (Karto.h:5810-5814);
 *                                  the caller reduces MIN on [0..1], MAX on [2..3] over the ranks
 *   2. b2s_occ_grid_create_shard -> grid dimensioned by the global box (ComputeDimensions, Karto.h:5816-5821),
 *                                  counters = this shard's rays; n_scans may be 0
 *   3. b2s_occ_grid_device_counters (all-reduce SUM on both) or b2s_occ_grid_set_counters (host arrays)
 *   4. b2s_occ_grid_update       -> cells from the summed counters (OccupancyGrid::Update, Karto.h:5953-5968) */
b2s_status b2s_occ_grid_scans_bbox(const b2s_laser *laser, int n_scans, const double *ranges, const double *poses,
                                   int device, void *cuda_stream, double bbox[4]);
b2s_status b2s_occ_grid_create_shard(const b2s_laser *laser, int n_scans, const double *ranges, const double *poses,
                                     double resolution, const double bbox[4], int device, void *cuda_stream,
                                     b2s_occ_grid **out);
b2s_status b2s_occ_grid_device_counters(b2s_occ_grid *g, uint32_t **d_pass, uint32_t **d_hit);
b2s_status b2s_occ_grid_set_counters(b2s_occ_grid *g, const uint32_t *pass, const uint32_t *hit);
/* step 3 with the collective inside the library: ncclAllReduce(SUM) of both counter planes in place through the caller's
 * ncclComm_t (dlopened libnccl.so.2), on the grid's stream */
b2s_status b2s_occ_grid_allreduce_counters(b2s_occ_grid *g, void *nccl_comm);
b2s_status b2s_occ_grid_update(b2s_occ_grid *g);
b2s_status b2s_occ_grid_info_get(const b2s_occ_grid *g, b2s_occ_grid_info *out);
/* cells: uint8 {0 unknown, 100 occupied, 255 free}; pass/hit: uint32 counters; any pointer may be NULL */
b2s_status b2s_occ_grid_copy(b2s_occ_grid *g, uint8_t *cells, uint32_t *pass, uint32_t *hit);
/* nav_msgs/OccupancyGrid payload as SlamKarto::updateMap fills it (karto_slam.cc:546-569):
 * int8 {-1,100,0}, row-major width x height (no width_step padding) */
b2s_status b2s_occ_grid_copy_ros(b2s_occ_grid *g, int8_t *out);
b2s_status b2s_occ_grid_last_timing(b2s_occ_grid *g, double out[2]); /* ms: ray-trace kernel, threshold kernel */
void b2s_occ_grid_destroy(b2s_occ_grid *g);

/* ---------------------------------------------------------------- K2a / K3: Hector log-odds grid map */

typedef struct b2s_hector_map b2s_hector_map; /* opaque: replaces hectorslam::GridMap (OccGridMapP) */

/* GridMap(mapResolution, size, offset) (GridMapBase.h:54-66, MapRepMultiMap.h:63-67): size x size cells,
 * start_x/start_y in [0,1] (fraction of the map at which the world origin sits). */
b2s_status b2s_hector_map_create(int size_x, int size_y, float resolution, float start_x, float start_y,
                                 int device, void *cuda_stream, b2s_hector_map **out);
void b2s_hector_map_destroy(b2s_hector_map *m);
/* GridMapLogOddsFunctions::setUpdateFreeFactor / setUpdateOccupiedFactor (GridMapLogOdds.h:116-134) */
b2s_status b2s_hector_map_set_factors(b2s_hector_map *m, float update_free, float update_occupied);
/* OccGridMapBase::updateByScan (OccGridMapBase.h:118-168): points are the DataContainer in map-cell units
 * ([n][2] float, already scaled by 1/resolution as hector_slam.cc:320-362 does), origo = sensor origin in the
 * same frame, pose = robot pose in WORLD coordinates (x, y, heading). */
b2s_status b2s_hector_map_update_by_scan(b2s_hector_map *m, const float *points, int n_points,
                                         const float origo[2], const float world_pose[3]);
/* OccGridMapBase::updateByScanJustOnce (OccGridMapBase.h:175-217), the make-map demo variant of lesson4
 * (hector_mapping/src/hector_mapping/...: map pose fixed at cell (800, 800), heading 0; points in METRES, the end cell is
 * begin + (int)round(p / 0.05)). */
b2s_status b2s_hector_map_update_by_scan_just_once(b2s_hector_map *m, const float *points, int n_points,
                                                   const float origo[2]);
/* ScanMatcher::matchData (ScanMatcher.h:60-98) on ONE grid level: Gauss-Newton scan-to-map alignment.
 * begin_world_pose in, new world pose + 3x3 Hessian ("covariance") out. */
b2s_status b2s_hector_map_match_data(b2s_hector_map *m, const float *points, int n_points,
                                     const float begin_world_pose[3], int max_iterations,
                                     float out_world_pose[3], float out_cov[9]);
/* raw cells: logOdds float + updateIndex int per cell (GridMapLogOdds.h:37-75) */
b2s_status b2s_hector_map_copy(b2s_hector_map *m, float *log_odds, int32_t *update_index);
/* nav_msgs/OccupancyGrid payload as HectorMappingRos::publishMap does (hector_slam.cc:254-317) */
b2s_status b2s_hector_map_copy_ros(b2s_hector_map *m, int8_t *out);
b2s_status b2s_hector_map_last_timing(b2s_hector_map *m, double out[2]);

/* ---------------------------------------------------------------- lesson4 front end: HectorSlamProcessor
 * One call per LaserScan = MapRepMultiMap::matchData (coarse-to-fine Gauss-Newton over all pyramid levels) + the
 * map-update gate + MapRepMultiMap::updateByScan (all levels) — all on the device: the processor's state (last poses,
 * update indices, the coarse levels' data containers) is device-resident, one cooperative launch does match + gate +
 * update, and the pose returns through a host-mapped mailbox as soon as the match is done.  A whole stream of scans can
 * be handed over at once (b2s_hector_slam_process_stream: no host round trip between scans), and a handle may hold B
 * independent processors (b2s_hector_slam_create_batch).
 * EXACT mode (default): bit-identical poses, Hessians and cells to the reference (sequential float32 sums in point
 * order, glibc's sinf / cosf restated on the device); b2s_hector_slam_set_exact(p, 0) sums with a tree instead and
 * spreads the per-point phase of the match over a 4-CTA cluster (faster; poses within 1e-4). */

typedef struct b2s_hector_slam b2s_hector_slam; /* opaque: replaces hectorslam::HectorSlamProcessor
                                                   (slam_main/HectorSlamProcessor.h:50-150) */

#define B2S_HECTOR_MAX_LEVELS 8

/* HectorSlamProcessor(mapResolution, mapSizeX, mapSizeY, startCoords, multi_res_size) (HectorSlamProcessor.h:56-65):
 * level l has cell length resolution * 2^l and size >> l cells; every level shares the level-0 offset
 * (MapRepMultiMap.h:56-89).  Defaults as the constructor sets them: update factors 0.4 / 0.6
 * (GridMapLogOdds.h:98-102), map-update gate 0.4 m / 0.13 rad. */
b2s_status b2s_hector_slam_create(float map_resolution, int map_size_x, int map_size_y, float start_x, float start_y,
                                  int levels, int device, void *cuda_stream, b2s_hector_slam **out);
void b2s_hector_slam_destroy(b2s_hector_slam *p);
/* setUpdateFactorFree / setUpdateFactorOccupied (HectorSlamProcessor.h:128-129) */
b2s_status b2s_hector_slam_set_update_factors(b2s_hector_slam *p, float update_free, float update_occupied);
/* setMapUpdateMinDistDiff / setMapUpdateMinAngleDiff (HectorSlamProcessor.h:130-131).  The gate is
 * util::poseDifferenceLargerThan (UtilFunctions.h:72-90), including its integer-truncating abs() on the angle. */
b2s_status b2s_hector_slam_set_map_update_min_diff(b2s_hector_slam *p, float min_dist, float min_angle);
/* reset() (HectorSlamProcessor.h:111-116): clears every level and the last poses */
b2s_status b2s_hector_slam_reset(b2s_hector_slam *p);
/* update(dataContainer, poseHintWorld, map_without_matching) (HectorSlamProcessor.h:81-108).  points = the
 * DataContainer in LEVEL-0 map-cell units ([n][2] float, as hector_slam.cc:320-362 fills it), origo likewise, pose
 * hint in world coordinates.  out_pose = getLastScanMatchPose(); out_cov (may be NULL) = getLastScanMatchCovariance()
 * (the level-0 Hessian; untouched when map_without_matching).  out_map_updated (may be NULL) tells whether the gate
 * let this scan into the maps. */
b2s_status b2s_hector_slam_update(b2s_hector_slam *p, const float *points, int n_points, const float origo[2],
                                  const float pose_hint_world[3], int map_without_matching, float out_pose[3],
                                  float out_cov[9], int *out_map_updated);
/* getMapLevels / getGridMap(level) (HectorSlamProcessor.h:124-125) */
b2s_status b2s_hector_slam_level_dims(b2s_hector_slam *p, int level, int dims[2], float *cell_length);
b2s_status b2s_hector_slam_copy_level(b2s_hector_slam *p, int level, float *log_odds, int32_t *update_index);
/* nav_msgs/OccupancyGrid payload of one level as HectorMappingRos::publishMap fills it (hector_slam.cc:254-317) */
b2s_status b2s_hector_slam_copy_level_ros(b2s_hector_slam *p, int level, int8_t *out);
/* out[0] = scans matched, out[1] = scans let into the maps, out[2] = Bresenham cell visits so far (all levels; summed
 * over the processors of a batched handle), out[3] / out[4] = ms of processor 0's last match / update (device timer) */
b2s_status b2s_hector_slam_stats(b2s_hector_slam *p, double out[5]);
/* 1 (default) = the reference's arithmetic bit for bit; 0 = the nine Gauss-Newton sums are tree-reduced instead of
 * accumulated in point order (everything else unchanged): faster, poses agree to ~1e-6 m */
b2s_status b2s_hector_slam_set_exact(b2s_hector_slam *p, int exact);
/* Non-exact mode, single-processor handles: the CTAs of one thread-block cluster share the per-point phase of every
 * Gauss-Newton iteration (pose out / nine partial sums back through distributed shared memory).  Returns the CTAs per
 * cluster in use: 4, or 1 (no cluster launch: one CTA matches) where the device or driver cannot co-schedule the grid
 * as clusters.  B2S_HS_CLUSTER=0 in the environment when the handle is created selects the one-CTA match on any device,
 * so that the two can be compared. */
int32_t b2s_hector_slam_match_cluster_size(const b2s_hector_slam *p);
/* The node's loop over a recorded stream (hector_slam.cc:195-204: update(container, getLastScanMatchPose())) in ONE
 * call: n_scans scans, points concatenated ([sum n_points][2], level-0 map-cell units), hint of scan i = pose of scan
 * i-1 (first_pose_hint for scan 0; NULL = the processor's current last scan-match pose), or pose_hints[i] when given
 * (required with map_without_matching).  out_poses [n_scans][3]; out_map_updated [n_scans] and out_last_cov[9] may be
 * NULL.  Identical results to n_scans b2s_hector_slam_update calls. */
b2s_status b2s_hector_slam_process_stream(b2s_hector_slam *p, int n_scans, const float *points, const int32_t *n_points,
                                          const float origo[2], const float *first_pose_hint, const float *pose_hints,
                                          int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                          float *out_last_cov);
/* B independent HectorSlamProcessors (robots / maps) behind one handle (SURVEY.md §8(e): Hector maps shard over
 * independent maps, not within one).  batch may be any count >= 1 whose maps fit in device memory (65 535 is not a
 * limit).  max_points = capacity of one scan (<= 4096). */
b2s_status b2s_hector_slam_create_batch(int batch, int max_points, float map_resolution, int map_size_x, int map_size_y,
                                        float start_x, float start_y, int levels, int device, void *cuda_stream,
                                        b2s_hector_slam **out);
/* update() of every processor with its own scan: points [B][max_points][2] (rows padded), n_points [B], pose_hints
 * [B][3] (NULL = each processor's last scan-match pose); out_poses [B][3], out_covs [B][9] / out_map_updated [B] may
 * be NULL. */
b2s_status b2s_hector_slam_update_batch(b2s_hector_slam *p, const float *points, const int32_t *n_points,
                                        const float origo[2], const float *pose_hints, int map_without_matching,
                                        float *out_poses, float *out_covs, int32_t *out_map_updated);
/* the same step on scans already in device memory (DEVICE pointers; asynchronous on the handle's stream, nothing
 * returned to the host; max_n = upper bound of n_points): the resident-in-HBM form */
b2s_status b2s_hector_slam_update_batch_device(b2s_hector_slam *p, const float *d_points, const int32_t *d_n_points,
                                               int max_n, const float origo[2], const float *d_pose_hints,
                                               int map_without_matching);
b2s_status b2s_hector_slam_sync(b2s_hector_slam *p);
b2s_status b2s_hector_slam_copy_level_of(b2s_hector_slam *p, int processor, int level, float *log_odds,
                                         int32_t *update_index);
/* nav_msgs/OccupancyGrid payload of one processor's level (b2s_hector_slam_copy_level_ros is processor 0's) */
b2s_status b2s_hector_slam_copy_level_ros_of(b2s_hector_slam *p, int processor, int level, int8_t *out);
/* b2s_hector_slam_process_stream for EVERY processor of the handle in one call, each over its own recording (any
 * handle, B = 1 included).  n_scans [B] (0: the processor is left untouched); scans are processor-major: processor b's
 * scans follow processor b-1's, n_points [sum n_scans] and the points ([sum n_points][2], level-0 map-cell units) in the
 * same order.  Hint of a processor's scan i = its pose of scan i-1 (first_pose_hints[b] for its first scan; NULL = its
 * current last scan-match pose), or pose_hints [sum n_scans][3] when given (required with map_without_matching).
 * out_poses [sum n_scans][3]; out_map_updated [sum n_scans] and out_last_covs [B][9] (the level-0 Hessian of the
 * processor's last scan; its row is untouched when it has no scans or with map_without_matching) may be NULL.
 * Processor b's poses, gate decisions, Hessian, last poses and cells are those of b2s_hector_slam_process_stream over
 * its scans on a single-processor handle with the same settings; two calls over consecutive parts of every recording
 * equal one.  ONE launch, one CTA per processor (nothing shared between them: B may exceed the resident CTAs).
 * Refused before anything is enqueued: B2S_ERR_BAD_PARAMS for NULL arrays or negative counts, B2S_ERR_TOO_LARGE for a
 * scan above the handle's max_points or a processor with 2^20 - 1 or more scans. */
b2s_status b2s_hector_slam_process_stream_batch(b2s_hector_slam *p, const int32_t *n_scans, const float *points,
                                                const int32_t *n_points, const float origo[2],
                                                const float *first_pose_hints, const float *pose_hints,
                                                int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                                float *out_last_covs);
/* One processor of a fleet handle: HectorSlamProcessor's constructor arguments (as for b2s_hector_slam_create) and
 * the values of its setters (b2s_hector_slam_set_update_factors, _set_map_update_min_diff).  The defaults of
 * b2s_hector_slam_create are update_free 0.4, update_occupied 0.6, min_dist 0.4 m, min_angle 0.13 rad.  reserved:
 * zero; it keeps the struct at 64 bytes. */
typedef struct b2s_hector_map_spec {
  float map_resolution;
  int32_t map_size_x, map_size_y;
  float start_x, start_y;
  int32_t levels;
  float update_free, update_occupied;
  float min_dist, min_angle;
  int32_t reserved[6];
} b2s_hector_map_spec;
/* B independent processors, each with its own map size, resolution, levels, start, update factors and map-update
 * gate (maps [batch]), behind one handle: b2s_hector_slam_create_batch with nothing required equal.  Every processor
 * gets its own planes (a processor with fewer levels has none above its last).  Each spec is checked as
 * b2s_hector_slam_create checks its arguments, before the device is touched, and the refusal names the processor:
 * B2S_ERR_BAD_PARAMS for levels outside 1 ... 8, a resolution that is not positive or a map whose coarsest level is
 * 2 cells or fewer across; B2S_ERR_TOO_LARGE for max_points above 4096.  process_stream_batch, process_scans_batch
 * (each processor scales the shared laser's points by its own level-0 cell length), update_batch and the _of getters
 * serve it; set_update_factors and set_map_update_min_diff set every processor's values.  b2s_hector_slam_create and
 * _create_batch are this with equal specs. */
b2s_status b2s_hector_slam_create_fleet(int batch, int max_points, const b2s_hector_map_spec *maps, int device,
                                        void *cuda_stream, b2s_hector_slam **out);
/* getGridMap(level) of one processor; B2S_ERR_BAD_PARAMS for a level at or above that processor's levels.
 * b2s_hector_slam_level_dims is processor 0's. */
b2s_status b2s_hector_slam_level_dims_of(b2s_hector_slam *p, int processor, int level, int dims[2], float *cell_length);
/* getLastScanMatchPose / getLastMapUpdatePose (HectorSlamProcessor.h:118-119) of one processor; either may be NULL */
b2s_status b2s_hector_slam_last_poses(b2s_hector_slam *p, int processor, float last_scan_match_pose[3],
                                      float last_map_update_pose[3]);
/* test hook: pretend `updates` map updates already consumed per-scan stamp epochs (exercises the 20-bit epoch wrap) */
b2s_status b2s_hector_slam_debug_set_epoch(b2s_hector_slam *p, unsigned int updates);

/* ---------------------------------------------------------------- ROS-shaped input adapters (host only; SURVEY.md §8(f).4)
 * The wire formats either side of the path: sensor_msgs/LaserScan in (here), nav_msgs/OccupancyGrid payloads out
 * (b2s_occ_grid_copy_ros, b2s_hector_map_copy_ros / b2s_hector_slam_copy_level_ros, b2s_gmap_copy_ros).  ROS itself is
 * out of scope; these are the conversions the lesson nodes perform on the message fields. */
typedef struct b2s_laser_scan_msg { /* the sensor_msgs/LaserScan fields the nodes read */
  float angle_min, angle_max, angle_increment, range_min, range_max;
  int32_t n_ranges;
  const float *ranges;
} b2s_laser_scan_msg;
/* SlamKarto::getLaser (lesson6/src/karto_slam.cc:323-395): the Custom LaserRangeFinder made from the first scan —
 * angles / ranges from the message, offset = laser pose in base_link (x, y, yaw), range threshold clipped into
 * [range_min, range_max] (Karto.h:3778-3787), n_readings = Round((max - min) / resolution) WITHOUT + 1
 * (LaserRangeFinder::Update, Karto.h:4152-4161).  Returns B2S_ERR_BAD_PARAMS if the message carries a different
 * number of ranges than that.  That check is this function's own, stricter than the reference: its
 * LaserRangeFinder::Validate(SensorData *) has the count comparison commented out (Karto.cpp:186-199) and accepts every
 * scan, and LocalizedRangeScan::Update then uses the first n_readings readings.  b2s_karto_node_create follows the
 * reference and accepts n_ranges >= n_readings. */
b2s_status b2s_ros_karto_laser(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                               b2s_laser *out);
/* SlamKarto::addScan (karto_slam.cc:407-434): float32 ranges -> kt_double readings, in reverse order for a laser
 * mounted upside-down (lasers_inverted_) */
b2s_status b2s_ros_karto_readings(const b2s_laser_scan_msg *scan, int inverted, double *out_readings);

/* ---------------------------------------------------------------- lesson6: the Karto SLAM node over whole recordings
 * SlamKarto (lesson6/src/karto_slam.cc) for one laser: its throttle, getLaser, getOdomPose, Mapper::Process (the device
 * Mapper, b2s_mapper_*), the map -> odom transform and the map-update gate with updateMap (the device occupancy grid,
 * b2s_occ_grid_*), over a recording handed in as arrays.  tests/test_karto_node_reference.py pins the restatement
 * oracle/karto_node_port.py to the unmodified node; tests/test_gpu_karto_node.py pins this handle to the restatement.
 * The tf arithmetic is tf's LinearMath in double, operation by operation (Transform product and inverse, Matrix3x3
 * setRotation / getRotation, Quaternion setRPY, getYaw through getRPY); ros::Time / Duration are roscpp's integer
 * arithmetic.  Neither tf nor roscpp is in the reference tree; the library's one definition of them (csrc/ros_math.cuh)
 * is held bit for bit to the node's stand-ins under oracle/shim/ by tests/test_ros_math.py (DESIGN.md §7). */
typedef struct b2s_karto_node_params {
  int32_t throttle_scans;     /* [1] a scan is processed when the count of scans handed in so far divides by it */
  int32_t reserved;           /* 0 */
  double map_update_interval; /* [5.0] s, ros::Duration::fromSec: a map is due when the stamp difference is STRICTLY
                                 greater */
  double resolution;          /* [0.05] m, OccupancyGrid::CreateFromScans */
  double use_scan_range;      /* [12.0] m, the laser's range threshold (clipped into [range_min, range_max]) */
  b2s_mapper_params mapper;   /* values as the Mapper STORES them after SlamKarto::InitParams (three of its setParam*
                                 calls square their argument); the matchers' range_threshold is replaced by the
                                 laser's */
} b2s_karto_node_params;

/* out_state values, one per scan handed in */
#define B2S_KARTO_THROTTLED 0    /* laser_count_ % throttle_scans != 0: the callback returned at once */
#define B2S_KARTO_NO_ODOM 1      /* the odom <- base_link lookup failed (a NaN in the scan's odom row): skipped */
#define B2S_KARTO_NOT_MOVED 2    /* Mapper::Process returned false (HasMovedEnough) */
#define B2S_KARTO_PROCESSED 3    /* Mapper::Process returned true */

/* One published map (the node's sst_.publish): info as b2s_occ_grid_info_get gives it (origin = offset, float32
 * resolution in the message = (float)resolution), payload [height][width] int8 as b2s_occ_grid_copy_ros.  scan_index
 * counts every scan handed to the handle, over all calls.  Both pointers are valid only during the call. */
typedef void (*b2s_karto_map_fn)(void *user, int32_t scan_index, const b2s_occ_grid_info *info, const int8_t *payload);

typedef struct b2s_karto_node b2s_karto_node; /* opaque: one SlamKarto */

/* SlamKarto's constructor and getLaser.  geometry = the recording's LaserScan fields (angle_min, angle_max,
 * angle_increment, range_min, range_max, n_ranges; its ranges pointer is not read).  The laser has m =
 * Round((angle_max - angle_min) / angle_increment) readings (LaserRangeFinder::Update, no + 1); a scan's first m
 * readings are used, after the reversal of an upside-down laser, and the rest are ignored, as the node does.  A standard
 * ROS scan (angle_max = angle_min + (n - 1) * angle_increment) has m = n - 1: its last beam is dropped.
 * laser_mount = base_link <- laser as translation xyz + quaternion xyzw: the laser's offset is its x, y and getYaw; it
 * is upside-down when the mount sends base_link's point (0, 0, 1 + z) to z <= 0 in the laser frame.  solver: NULL =
 * use_back_end false (the node's default), else the back end Mapper::SetScanSolver gets (copied; its user data must
 * outlive the handle).  B2S_ERR_BAD_PARAMS for NULL pointers, throttle_scans <= 0 (the node divides by it),
 * resolution not > 0, a map_update_interval that is not finite or outside ros::Duration's 32-bit range, a zero
 * angle_increment, a zero / non-finite mount quaternion, m < 1, or n_ranges < m (the node reads past the message's
 * ranges); whatever b2s_mapper_create refuses; B2S_ERR_NO_DEVICE without a device. */
b2s_status b2s_karto_node_create(const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                                 const double laser_mount[7], const b2s_scan_solver *solver, int device,
                                 b2s_karto_node **out);
void b2s_karto_node_destroy(b2s_karto_node *node);
/* The inner Mapper: b2s_mapper_get_poses / _get_edges / _stats / _scan_count read the node's graph.  Owned by the
 * node; do not destroy it or process scans through it. */
b2s_mapper *b2s_karto_node_mapper(b2s_karto_node *node);
/* SlamKarto::laserCallback on the next n_scans LaserScans: ranges [n_scans][n_ranges] float32 (widened to double as the
 * node does), stamps [n_scans][2] = header.stamp (sec, nsec), odom [n_scans][7] = the odom <- base_link transform the
 * tf lookup answers at that stamp (translation xyz + quaternion xyzw; any NaN = the lookup fails).  Per scan:
 * out_state (B2S_KARTO_*), out_pose [3] the corrected pose Mapper::Process left (0 unless processed), out_map_to_odom
 * [7] map_to_odom_ after the scan (translation xyz + quaternion xyzw, from getRotation), out_map_published 1 when
 * updateMap published; any output may be NULL.  A processed scan's scan time is 0 (the node never sets it), so
 * minimum_time_interval never admits a scan.  A map is built when none was yet or the stamp minus the last map's stamp
 * exceeds map_update_interval, from every processed scan at its corrected pose at that moment (they move after a loop
 * closure when a solver is set), and handed to on_map (may be NULL) before the call goes on.  Two calls over
 * consecutive parts of a recording equal one call.  B2S_ERR_BAD_PARAMS (nothing written) for NULL arrays with
 * n_scans > 0 or n_scans < 0; B2S_ERR_BAD_STATE after a call failed inside the Mapper (its rows up to the failing scan
 * are written then).  Returns when every map has been handed out. */
b2s_status b2s_karto_node_process(b2s_karto_node *node, int n_scans, const float *ranges, const uint32_t *stamps,
                                  const double *odom, int32_t *out_state, double *out_pose, double *out_map_to_odom,
                                  int32_t *out_map_published, b2s_karto_map_fn on_map, void *user);

/* Several nodes per handle, one per recording or per setting.  Each node runs its own Mapper, unchanged, on a worker
 * thread of its own for the length of a call; its device work (each MatchScan batch, each map build) is a request to
 * the calling thread, which serves the requests of all nodes in rounds: round k holds the k-th request of every node
 * still running, so the rounds follow from the data, not from thread timing.  A round's matches go out grouped by
 * matcher and search kind on two matcher handles shared by all nodes (each node's scans in their device pools once),
 * and its maps are built in one b2s_occ_grid_create_from_scans_batch over float32 readings the handle keeps on the
 * device (each uploaded once).  Every node equals its own b2s_karto_node_create handle bit for bit: states, poses,
 * map_to_odom, graph, b2s_mapper_stats and maps.  Threads are created by each call and joined before it returns.
 * A node's solver callbacks run on its worker thread, concurrently with the other nodes' workers, so a solver instance
 * must serve one node only.  b2s_karto_node_create is this with batch = 1; on a handle with batch > 1
 * b2s_karto_node_process answers B2S_ERR_BAD_PARAMS and b2s_karto_node_mapper NULL. */

/* b2s_karto_map_fn with the node the map belongs to; scan_index counts that node's scans */
typedef void (*b2s_karto_node_batch_map_fn)(void *user, int32_t node, int32_t scan_index, const b2s_occ_grid_info *info,
                                            const int8_t *payload);

/* params [batch], laser_mounts [batch][7], solvers [batch] or NULL (no back end for any node; a slot whose compute is
 * NULL: none for that node).  Each node is validated as b2s_karto_node_create validates its own, the refusal naming
 * the node.  All nodes share one geometry, one laser and two matchers: the laser getLaser derives (offset, range
 * threshold, upside-down flag) and mapper.sequential / mapper.loop after their range_threshold is replaced must be equal
 * bit for bit in every node, else B2S_ERR_BAD_PARAMS (two mounts may differ where the laser does not, e.g. in z).
 * throttle_scans, map_update_interval, resolution, the Mapper's host-only fields (travel gates, buffer size, link and
 * loop thresholds, do_loop_closing, ...) and the solver may differ.  B2S_ERR_TOO_LARGE for more than 1024 nodes. */
b2s_status b2s_karto_node_create_batch(int batch, const b2s_karto_node_params *params, const b2s_laser_scan_msg *geometry,
                                       const double *laser_mounts, const b2s_scan_solver *solvers, int device,
                                       b2s_karto_node **out);
/* node b's Mapper (0 <= b < batch), for the getters as b2s_karto_node_mapper; NULL out of range */
b2s_mapper *b2s_karto_node_mapper_of(b2s_karto_node *node, int b);
/* b2s_karto_node_process on every node at once: n_scans [batch] (0 leaves a node untouched), ranges / stamps / odom
 * and the outputs node-major (node 0's scans first).  Each node's maps reach on_map in its own order; across nodes
 * they arrive round by round, inside a round by ascending node, the same for the same calls.  Two calls over
 * consecutive parts of every recording, split anywhere per node, equal one call.  B2S_ERR_BAD_PARAMS (nothing written,
 * nothing changed) for a NULL n_scans, a negative count or NULL arrays with scans; B2S_ERR_BAD_STATE after a failed
 * call.  A device error or a Mapper failure in any node stops every node at its next request; the call returns the
 * first failure (lowest round, then lowest node), named in b2s_last_error(), each node's rows up to its stop are
 * written, and the handle refuses later calls with B2S_ERR_BAD_STATE. */
b2s_status b2s_karto_node_process_batch(b2s_karto_node *node, const int32_t *n_scans, const float *ranges,
                                        const uint32_t *stamps, const double *odom, int32_t *out_state, double *out_pose,
                                        double *out_map_to_odom, int32_t *out_map_published,
                                        b2s_karto_node_batch_map_fn on_map, void *user);
/* Where the last process call went: out[0] rounds, out[1] matcher launches, out[2] matches, out[3] maps built,
 * out[4] s serving matches, out[5] s building maps (both host wall time on the calling thread, device work included),
 * out[6] bytes the map builds copied back from the device, out[7] s of the whole call */
b2s_status b2s_karto_node_last_timing(const b2s_karto_node *node, double out[8]);
/* HectorMappingRos::rosPointCloudToDataContainer (lesson4/src/hector_mapping/hector_slam.cc:320-362): laser-frame points
 * ([n][3] float x, y, z as laser_geometry projected them) -> DataContainer entries in map-cell units.  laser_in_base =
 * (x, y, z, yaw) of the laser in base_link.  Filters: squared distance in (min_dist^2, max_dist^2), not behind the robot
 * within 0.5 m^2, not beyond use_max_scan_range, height window (z_min, z_max).  out_points [n][2] (capacity n),
 * out_origo[2] = laser position * scale_to_map.  Returns the number of points kept in *out_n. */
b2s_status b2s_ros_hector_points(const float *points_xyz, int n, const float laser_in_base[4], float scale_to_map,
                                 float min_dist, float max_dist, double use_max_scan_range, float z_min, float z_max,
                                 float *out_points, float out_origo[2], int32_t *out_n);
/* The settings of HectorMappingRos::scanCallback (lesson4/src/hector_mapping/hector_slam.cc:186-205) for turning raw
 * LaserScan ranges into a DataContainer: laser_geometry's projectLaser(scan, cloud, range_cutoff), then
 * rosPointCloudToDataContainer with the node's parameters.  Node defaults (hector_slam.cc:129, 150-161) in brackets. */
typedef struct b2s_hector_scan_filter {
  float laser_in_base[4];     /* x, y, z, yaw of the laser in base_link */
  double range_cutoff;        /* [30.0] projectLaser keeps range < range_cutoff && range >= range_min; < 0: range_max */
  double use_max_scan_range;  /* [20.0] */
  float min_dist, max_dist;   /* [0.2, 30.0] squared-distance window */
  float z_min, z_max;         /* [-1, 1] height window (the projected z is 0) */
} b2s_hector_scan_filter;
/* HectorMappingRos::scanCallback's conversion of n_scans LaserScans of one laser: geometry gives angle_min,
 * angle_increment, range_min, range_max and n_ranges (its ranges pointer is ignored); ranges [n_scans][n_ranges] float32.
 * Beam i projects along (cos, sin)(angle_min + i * angle_increment) computed in double, x / y = (float)(range * unit),
 * z = 0, then passes b2s_ros_hector_points' filters and transform.  out_points [sum out_n_points][2] are the kept
 * beams of every scan, in beam order, packed scan after scan (capacity n_scans * n_ranges): the input of
 * b2s_hector_slam_process_stream_batch, or with n_scans = 1 of b2s_hector_slam_update.  out_n_points [n_scans];
 * out_origo[2] = laser position * scale_to_map (scale_to_map = 1 / level-0 cell length, GridMapBase::getScaleToMap). */
b2s_status b2s_ros_hector_scans(const b2s_laser_scan_msg *geometry, const b2s_hector_scan_filter *filter, float scale_to_map,
                                int n_scans, const float *ranges, float *out_points, int32_t *out_n_points,
                                float out_origo[2]);
/* b2s_hector_slam_process_stream_batch on raw ranges: every processor of the handle walks its own recording of
 * LaserScans of ONE laser (geometry + filter as for b2s_ros_hector_scans, scale_to_map = the handle's level-0 1 / cell
 * length, origo = laser position * scale_to_map), converted on the device inside the same launch.  n_scans [B]
 * (processor-major recordings, 0 = untouched), ranges [sum n_scans][geometry->n_ranges] float32; hints, outputs and
 * the per-processor results as for b2s_hector_slam_process_stream_batch fed b2s_ros_hector_scans' points, which they
 * equal bit for bit.  out_n_points [sum n_scans] (may be NULL): the beams each scan kept.
 * Refused before anything is enqueued: B2S_ERR_BAD_PARAMS for NULL arrays or negative counts, B2S_ERR_TOO_LARGE for
 * n_ranges above the handle's max_points or a processor with 2^20 - 1 or more scans. */
b2s_status b2s_hector_slam_process_scans_batch(b2s_hector_slam *p, const b2s_laser_scan_msg *geometry,
                                               const b2s_hector_scan_filter *filter, const int32_t *n_scans,
                                               const float *ranges, const float *first_pose_hints, const float *pose_hints,
                                               int map_without_matching, float *out_poses, int32_t *out_map_updated,
                                               float *out_last_covs, int32_t *out_n_points);

/* ---------------------------------------------------------------- lesson4: the Hector SLAM node over whole recordings
 * HectorMappingRos (lesson4/src/hector_mapping/hector_slam.cc) for one laser: InitParams, the LaserScan conversion with
 * the full laser mount, HectorSlamProcessor::update (the device processor, b2s_hector_slam_*), the pose-info message and
 * tf (PoseInfoContainer.h) and publishMap of level 0 with its update-index gate, over a recording handed in as arrays.
 * tests/test_gpu_hector_node.py pins this handle to the restatement oracle/hector_node_port.py.
 *
 * The publish schedule is the library's own (the node publishes from a thread every map_pub_period of wall time, so the
 * reference's schedule depends on thread timing; DESIGN.md §7): tick 0 is the stamp of the first scan ever handed in,
 * tick k = tick 0 + k * Duration::fromSec(map_pub_period) in roscpp's integer arithmetic.  Before scan i is processed,
 * if its stamp >= the next tick, the map is published once, stamped with that tick, and the next tick becomes the first
 * tick strictly after scan i's stamp (no catch-up over gaps).  So map 0 precedes scan 0 and is all -1, as the node's
 * first publish at construction is. */
typedef struct b2s_hector_node_params { /* HectorMappingRos::InitParams (hector_slam.cc:119-162), node defaults [] */
  double map_resolution;             /* [0.05] m, cast to float for the processor */
  int32_t map_size;                  /* [2048] cells, square */
  int32_t map_multi_res_levels;      /* [3] */
  double map_start_x, map_start_y;   /* [0.5, 0.5] cast to float */
  double update_factor_free;         /* [0.4] (float setter) */
  double update_factor_occupied;     /* [0.9] */
  double map_update_distance_thresh; /* [0.4] */
  double map_update_angle_thresh;    /* [0.9] */
  double use_max_scan_range;         /* [20.0] m */
  double laser_min_dist;             /* [0.2] m; the handle squares it in double, then rounds to float, as the node */
  double laser_max_dist;             /* [30.0] m; likewise */
  float laser_z_min_value;           /* [-1.0] */
  float laser_z_max_value;           /* [1.0] */
  double map_pub_period;             /* [2.0] s */
} b2s_hector_node_params;

/* nav_msgs/MapMetaData as setMapInfo fills it (hector_slam.cc:165-180): origin = getWorldCoords(0, 0) - cell length / 2
 * (float, widened), orientation identity, resolution = the float cell length, width / height = level 0's size */
typedef struct b2s_hector_node_map_info {
  double origin_x, origin_y;
  float resolution;
  int32_t width, height;
} b2s_hector_node_map_info;

/* One published map: scan_index = the scans handed to the handle before it (over all calls), stamp (sec, nsec) = its
 * tick (or the stamp given to b2s_hector_node_publish_map), payload [height][width] int8 (-1 / 0 / 100), rebuilt = 1
 * when the grid's update index differed from the one at the previous publish (publishMap's gate; the payload is the
 * same bytes either way).  Pointers are valid only during the call. */
typedef void (*b2s_hector_node_map_fn)(void *user, int32_t scan_index, const uint32_t stamp[2],
                                       const b2s_hector_node_map_info *info, const int8_t *payload, int32_t rebuilt);

typedef struct b2s_hector_node b2s_hector_node; /* opaque: one HectorMappingRos */

/* The node's constructor.  geometry = the recording's LaserScan fields (angle_min, angle_increment, range_min,
 * range_max, n_ranges; its ranges pointer is not read); projectLaser's cutoff is 30 m as in the node.  laser_mount =
 * base_link <- laser, translation xyz + quaternion xyzw (what the listener answers in the constructor); its basis is
 * Matrix3x3::setRotation of the quaternion.  B2S_ERR_BAD_PARAMS for NULL pointers, a zero or non-finite mount, a
 * non-positive resolution or map size, levels the processor refuses, a map_pub_period that is not positive and finite or
 * whose ros::Duration is zero or outside its 32-bit range, and a zero angle_increment; B2S_ERR_TOO_LARGE for n_ranges
 * above 4096; B2S_ERR_NO_DEVICE without a device. */
b2s_status b2s_hector_node_create(const b2s_hector_node_params *params, const b2s_laser_scan_msg *geometry,
                                  const double laser_mount[7], int device, b2s_hector_node **out);
void b2s_hector_node_destroy(b2s_hector_node *node);
/* The inner processor: b2s_hector_slam_level_dims / _copy_level / _copy_level_ros / _last_poses / _stats read the
 * node's maps and poses.  Owned by the node; do not destroy it or process scans through it.  The node always runs in
 * exact mode. */
b2s_hector_slam *b2s_hector_node_processor(b2s_hector_node *node);
/* HectorMappingRos::scanCallback on the next n_scans LaserScans: ranges [n_scans][n_ranges] float32, stamps
 * [n_scans][2] = header.stamp (sec, nsec).  Per scan (any output may be NULL):
 *   out_pose [3] float        getLastScanMatchPose after the scan
 *   out_pose_msg [7] double   the PoseWithCovarianceStamped pose: x, y, 0, 0, 0, sin(yaw * 0.5f), cos(yaw * 0.5f)
 *                             (the double sin / cos of the float half angle, as the node's unqualified calls bind
 *                             under the stand-in headers; DESIGN.md §7).  odom_hector carries the same pose; the
 *                             odom -> base_link tf is poseMsgToTF of it, and map -> odom stays the identity.
 *   out_cov [36] double       lastScanMatchCov (the level-0 Hessian) spread as PoseInfoContainer::update does, every
 *                             other entry 0.  A scan that keeps no beams leaves lastScanMatchCov as it was; before the
 *                             first matched scan the node reads an uninitialised matrix, and the handle reports zeros.
 *   out_map_updated           the gate's map-update decision
 *   out_n_points              the beams the conversion kept
 * Maps due by the schedule go to on_map (may be NULL) before the call returns, in order.  Two calls over consecutive
 * parts of a recording equal one call.  B2S_ERR_BAD_PARAMS (nothing written, nothing changed) for NULL arrays with
 * n_scans > 0 or n_scans < 0; B2S_ERR_TOO_LARGE for 2^20 - 1 or more scans in one call.  A call that fails after it
 * started (a CUDA error) may already have handed out maps and moved the processor; the handle then answers every
 * later process / publish_map call with B2S_ERR_BAD_STATE and must be destroyed. */
b2s_status b2s_hector_node_process(b2s_hector_node *node, int n_scans, const float *ranges, const uint32_t *stamps,
                                   float *out_pose, double *out_pose_msg, double *out_cov, int32_t *out_map_updated,
                                   int32_t *out_n_points, b2s_hector_node_map_fn on_map, void *user);
/* The node's publishMap of level 0 now, stamped `stamp` (sec, nsec): for a caller with its own clock and for the final
 * map.  It shares the update-index gate with the scheduled publishes and does not move the schedule. */
b2s_status b2s_hector_node_publish_map(b2s_hector_node *node, const uint32_t stamp[2], b2s_hector_node_map_fn on_map,
                                       void *user);

/* Several nodes per handle, one per recording or per setting, run side by side on the device (one CTA per node).
 * b2s_hector_node_create is this with batch = 1; on a handle with batch > 1, b2s_hector_node_process and
 * b2s_hector_node_publish_map answer B2S_ERR_BAD_PARAMS.  b2s_hector_node_processor returns the batched processor:
 * its _of getters read node b. */

/* b2s_hector_node_map_fn with the node the map belongs to; scan_index counts that node's scans */
typedef void (*b2s_hector_node_batch_map_fn)(void *user, int32_t node, int32_t scan_index, const uint32_t stamp[2],
                                             const b2s_hector_node_map_info *info, const int8_t *payload,
                                             int32_t rebuilt);

/* params [batch], laser_mounts [batch][7]: one set per node, validated as b2s_hector_node_create validates its own
 * (the refusal names the node).  The fields the processor holds once (map_resolution, map_size,
 * map_multi_res_levels, map_start_x / _y, update_factor_free / _occupied, map_update_distance_thresh / _angle_thresh)
 * must be equal in every set, else B2S_ERR_BAD_PARAMS; the mount, laser_min_dist / _max_dist, use_max_scan_range, the
 * z window and map_pub_period may differ.  All nodes share one geometry.  B2S_ERR_TOO_LARGE for more than 65535 nodes. */
b2s_status b2s_hector_node_create_batch(int batch, const b2s_hector_node_params *params,
                                        const b2s_laser_scan_msg *geometry, const double *laser_mounts, int device,
                                        b2s_hector_node **out);
/* Nodes of different robots in one handle: params [batch], geometries [batch] (each node's own LaserScan fields) and
 * laser_mounts [batch][7], nothing required equal.  Each node gets its own processor (map size, resolution, levels,
 * start, update factors, map-update gate) and its own laser, and is validated as b2s_hector_node_create validates its
 * own, before the device is touched; the refusal names the node (B2S_ERR_TOO_LARGE for n_ranges above 4096 or more
 * than 65535 nodes).  b2s_hector_node_create_batch is this with one geometry repeated.  process_batch reads node b's
 * n_scans[b] scans as rows of its own n_ranges floats, node-major; each map carries its node's map info and payload
 * size. */
b2s_status b2s_hector_node_create_fleet(int batch, const b2s_hector_node_params *params,
                                        const b2s_laser_scan_msg *geometries, const double *laser_mounts, int device,
                                        b2s_hector_node **out);
/* b2s_hector_node_process on every node at once: n_scans [batch] (0 leaves a node untouched, its schedule does not
 * start), ranges / stamps / outputs node-major (node 0's scans first), as b2s_hector_slam_process_scans_batch.  Each
 * node's maps reach on_map in its own publish order.  Across nodes the call runs in parts: part 0 holds every node's
 * scans before its first publish in the call, part k >= 1 starts with the k-th publish of every node that has one; maps
 * arrive part by part, and inside a part by ascending node.  Two calls over consecutive parts of every recording equal
 * one call.  B2S_ERR_BAD_PARAMS (nothing written, nothing changed) for a NULL n_scans, a negative count, or NULL
 * arrays with scans; B2S_ERR_TOO_LARGE for a node with 2^20 - 1 or more scans.  A failure after the call started marks
 * the handle failed, as for b2s_hector_node_process.  The maps due before a part are converted on the device into one
 * page-locked buffer per part, two parts in flight: 2 x (the most cells published before one part) bytes on each
 * side, allocated by the first call that publishes and kept (grown by a later call that publishes more). */
b2s_status b2s_hector_node_process_batch(b2s_hector_node *node, const int32_t *n_scans, const float *ranges,
                                         const uint32_t *stamps, float *out_pose, double *out_pose_msg, double *out_cov,
                                         int32_t *out_map_updated, int32_t *out_n_points,
                                         b2s_hector_node_batch_map_fn on_map, void *user);
/* b2s_hector_node_publish_map of node b (0 <= b < batch): shares node b's update-index gate, leaves the others' */
b2s_status b2s_hector_node_publish_map_of(b2s_hector_node *node, int b, const uint32_t stamp[2],
                                          b2s_hector_node_batch_map_fn on_map, void *user);

/* ---------------------------------------------------------------- K2b: GMapping hit/visit map */

typedef struct b2s_gmap b2s_gmap; /* opaque: replaces GMapping::ScanMatcherMap (gmapping.cc:135) */

/* ScanMatcherMap(center, xmin, ymin, xmax, ymax, delta) (map.h:117-140): note the (cells >> 5) patch rounding. */
b2s_status b2s_gmap_create(double center_x, double center_y, double xmin, double ymin, double xmax, double ymax,
                           double delta, int device, void *cuda_stream, b2s_gmap **out);
void b2s_gmap_destroy(b2s_gmap *g);
b2s_status b2s_gmap_size(const b2s_gmap *g, int32_t size_xy[2]);
/* GMapping::ComputeMap (gmapping.cc:171-242) for one scan: ranges[n], angles[n] (beam angles in the laser
 * frame), laser pose in world, max_range / max_urange. */
b2s_status b2s_gmap_compute_map(b2s_gmap *g, const double *ranges, const double *angles, int n,
                                const double laser_pose[3], double max_range, double max_urange);
/* PointAccumulator per cell (map.h:17-48): n, visits, acc.x, acc.y */
b2s_status b2s_gmap_copy(b2s_gmap *g, int32_t *n, int32_t *visits, float *acc_x, float *acc_y);
/* the published map (gmapping.cc:141-159): -1 unknown, 100 if n/visits > 0.25 else 0 */
b2s_status b2s_gmap_copy_ros(b2s_gmap *g, int8_t *out);

/* ---------------------------------------------------------------- K3 (lesson3): PL-ICP fine alignment */

/* The subset of CSM's sm_params the reference sets (lesson3/src/plicp_odometry.cc:72-185), defaults in comments. */
typedef struct b2s_icp_params {
  double max_angular_correction_deg; /* 45 */
  double max_linear_correction;      /* 1.0 m (the node's yaml default; CSM's is 0.5) */
  double epsilon_xy;                 /* 1e-6 */
  double epsilon_theta;              /* 1e-6 */
  double max_correspondence_dist;    /* 1.0 m */
  double outliers_maxPerc;           /* 0.90 */
  double outliers_adaptive_order;    /* 0.7 */
  double outliers_adaptive_mult;     /* 2.0 */
  int32_t max_iterations;            /* 10 */
  int32_t use_point_to_line_distance;/* 1 */
  int32_t outliers_remove_doubles;   /* 1 */
  int32_t reserved;
} b2s_icp_params;

typedef struct b2s_icp_result {
  double x[3];        /* sm_result.x: pose of the current scan in the reference scan's frame (plicp_odometry.cc:399-403).
                         When valid = 0 it is the last accepted estimate, or first_guess if no iteration succeeded —
                         never the output of the iteration that failed (too few correspondences, or a solve without a
                         finite solution) */
  double error;       /* sum of point-to-segment distances of the kept correspondences */
  int32_t valid;      /* sm_result.valid */
  int32_t iterations; /* iterations that succeeded; the one that failed is not counted */
  int32_t nvalid;     /* correspondences kept in the last iteration, the failed one included */
  int32_t reserved;
} b2s_icp_result;

/* sm_icp (plicp_odometry.cc:391) for `batch` independent scan pairs: ref_ranges / sens_ranges [batch][n] on the beam
 * angles theta[n] (LaserScanToLDP, :285-322: a reading is valid iff range_min < r < range_max), first_guess [batch][3].
 * PARITY UNPINNED: CSM is an external, un-versioned dependency absent from the reference tree; this follows the
 * published algorithm (Censi, ICRA 2008) — see DESIGN.md §7. */
b2s_status b2s_plicp_match(const b2s_icp_params *params, int batch, int n, const double *ref_ranges,
                           const double *sens_ranges, const double *theta, double range_min, double range_max,
                           const double *first_guess, int device, void *cuda_stream, b2s_icp_result *results);

/* ScanMatchPLICP (lesson3/src/plicp_odometry.cc:191-517), the node around sm_icp, for B independent recordings (robots)
 * (each of its own laser, mount and parameters with b2s_plicp_odom_create_fleet): key frame, constant-velocity prediction (GetPrediction, :442-456: only linear.x >= 1e-6 predicts; there
 * is never an angular prediction), the prediction moved into the laser frame through the base-to-laser transform,
 * sm_icp against the key frame (the matcher of b2s_plicp_match), the correction composed into base_in_odom_ and the
 * key-frame rule (NewKeyframeNeeded, :498-517: |yaw| > kf_dist_angular, then ++count == kf_scan_count, which alone
 * resets the count, then x^2 + y^2 > kf_dist_linear^2).  The state is the node's: tf2::Transform (3x3 basis and origin
 * in double) for base_in_odom_ and base_in_odom_keyframe_, latest_velocity_, last_icp_time_, the scan count and the key
 * frame's float32 ranges.  dt = (stamp - last stamp) as ros::Time arithmetic; equal stamps give dt = 0 and an inf / NaN
 * velocity, kept as IEEE arithmetic gives it.  last_icp_time_ always advances; velocity and pose change only on a valid
 * match.  Each LaserScan is converted with its own message's range fields (LaserScanToLDP, :285-322); the key frame
 * keeps the valid flags its own message gave it (prev_ldp_scan_), so the handle keeps its fields with its ranges.  One rule the node leaves undefined: after a failed match (icp.valid = 0) the node tests the key-frame rule on
 * a default-constructed, uninitialised tf2::Transform; here it is the identity, so only the scan-count rule can
 * promote such a scan (DESIGN.md §7).  Pinned to the unmodified node except sm_icp and tf2's LinearMath, whose
 * published code is restated (PARITY UNPINNED for sm_icp; the device's sin / cos / atan2 may differ from glibc's in the
 * last place). */
typedef struct b2s_plicp_odom_params {
  b2s_icp_params icp;              /* sm_params subset, node defaults (b2s_icp_params) */
  double kf_dist_linear;           /* 0.1 m */
  double kf_dist_angular;          /* 5 deg, in rad */
  int32_t kf_scan_count, reserved; /* 10 */
  double base_to_laser[7];         /* translation x, y, z + quaternion x, y, z, w: lookupTransform(base, laser) */
} b2s_plicp_odom_params;

typedef struct b2s_plicp_odom_step { /* one LaserScan's outcome */
  double position[3], orientation[4]; /* odom_msg.pose.pose = toMsg(base_in_odom_) (orientation x, y, z, w) */
  double linear[3], angular[3];       /* odom_msg.twist.twist = latest_velocity_ */
  double first_guess[3];              /* input_.first_guess */
  b2s_icp_result icp;                 /* output_ */
  int32_t published;      /* 0 for a recording's first scan (initialisation only: nothing published, all fields 0
                             except orientation w = 1, keyframe = 1, reference_scan = -1) */
  int32_t keyframe;       /* this scan became the key frame */
  int32_t reference_scan; /* index in the recording of the key frame it was matched against */
  int32_t reserved;
} b2s_plicp_odom_step;

typedef struct b2s_plicp_odom b2s_plicp_odom; /* opaque: B ScanMatchPLICP nodes */

/* The LaserScan fields the node reads per recording (LaserScanToLDP, :285-322), fixed for a recording at create. */
typedef struct b2s_plicp_odom_laser { /* 16 bytes */
  int32_t n_beams;                    /* scan_msg->ranges.size() */
  float angle_min, angle_increment;   /* float32 message fields; beam i at angle_min + i * angle_increment summed in
                                         float (:308), then widened */
  int32_t reserved;                   /* 0 */
} b2s_plicp_odom_laser;

/* B ScanMatchPLICP nodes, one per recording: recording b has its own params[b] (sm_params subset, key-frame thresholds,
 * base_to_laser mount, :64-185 and GetBaseToLaserTf :257-280) and its own lasers[b].  Range fields are per scan
 * (b2s_plicp_odom_process_fleet).  Pinned to the unmodified node except sm_icp and tf2's LinearMath (PARITY UNPINNED for
 * sm_icp, see above).  Everything is checked before the device is touched: B2S_ERR_BAD_PARAMS for NULL pointers,
 * batch < 1, n_beams < 3, icp.max_iterations < 1, a zero / non-finite mount quaternion or a non-zero laser reserved,
 * the refusal naming the recording in b2s_last_error(); B2S_ERR_NO_DEVICE without a device; B2S_ERR_TOO_LARGE when a
 * recording is above the pair kernel's beam limit (2408 on an H100, 82 bytes of shared memory per beam). */
b2s_status b2s_plicp_odom_create_fleet(int batch, const b2s_plicp_odom_params *params /* [batch] */,
                                       const b2s_plicp_odom_laser *lasers /* [batch] */, int device, void *cuda_stream,
                                       b2s_plicp_odom **out);
/* One laser geometry, one parameter set and fixed range fields for every recording: the fleet of `batch` equal rows
 * whose scans all carry range_min, range_max (valid iff range_min < r < range_max, :295).  Refusals as
 * b2s_plicp_odom_create_fleet's. */
b2s_status b2s_plicp_odom_create(const b2s_plicp_odom_params *params, int batch, int n_beams, float angle_min,
                                 float angle_increment, float range_min, float range_max, int device, void *cuda_stream,
                                 b2s_plicp_odom **out);
void b2s_plicp_odom_destroy(b2s_plicp_odom *h);
/* ScanCallback on every recording's next n_scans[b] LaserScans (0: recording b is untouched), in ONE launch (one CTA per
 * recording, no host round trip between scans).  Recordings are processor-major and ragged: ranges holds n_scans[0]
 * scans of n_beams[0] floats, then n_scans[1] scans of n_beams[1] floats, ...; range_limits [sum n_scans][2] = each
 * scan's float32 (range_min, range_max); stamps [sum n_scans][2] (header.stamp sec, nsec); out [sum n_scans].  Works on
 * handles of both create functions.  Two calls over consecutive parts of every recording, cut anywhere per recording,
 * equal one call.  Refused before anything is enqueued or written, every recording's state unchanged:
 * B2S_ERR_BAD_PARAMS for a NULL n_scans, a negative count or NULL arrays when the call has scans; B2S_ERR_TOO_LARGE for
 * more than 2^31 - 1 scans. */
b2s_status b2s_plicp_odom_process_fleet(b2s_plicp_odom *h, const int32_t *n_scans, const float *ranges,
                                        const float *range_limits, const uint32_t *stamps, b2s_plicp_odom_step *out);
/* b2s_plicp_odom_process_fleet with the create-time range fields for every scan: ranges [sum n_scans][n_beams].
 * B2S_ERR_BAD_PARAMS on a handle from b2s_plicp_odom_create_fleet (it has no create-time fields). */
b2s_status b2s_plicp_odom_process(b2s_plicp_odom *h, const int32_t *n_scans, const float *ranges, const uint32_t *stamps,
                                  b2s_plicp_odom_step *out);
/* a fresh node for one recording, or for all with recording = -1: its next scan initialises it */
b2s_status b2s_plicp_odom_reset(b2s_plicp_odom *h, int recording);

/* ScanMatchPLICP (lesson3/src/scan_match_plicp.cc:162-300), lesson3's scan-to-scan node, for B independent recordings,
 * each of its own laser: every LaserScan is converted to an LDP (LaserScanToLDP, :220-261: valid iff range_min < r <
 * range_max with the message's own float32 fields, so NaN and +-inf are invalid; beam angle angle_min + i *
 * angle_increment summed in float) and matched by sm_icp (the matcher of b2s_plicp_match) against the scan before it
 * from a zero first guess; the new scan then becomes the previous one.  The pairs of a recording are independent, so a
 * call runs ONE launch with one CTA per scan pair across all recordings.  Pinned to the unmodified node except sm_icp
 * (PARITY UNPINNED, DESIGN.md §7). */
typedef struct b2s_plicp_scan_match_step { /* one LaserScan's outcome */
  b2s_icp_result icp; /* output_ (all zero when matched = 0) */
  double theta_deg;   /* output_.x[2] * 180 / M_PI in the node's operation order (what it prints, :289), valid or not */
  int32_t matched;    /* 0 for the scan that initialises the node (nothing matched), else 1 */
  int32_t reserved;
} b2s_plicp_scan_match_step;

typedef struct b2s_plicp_scan_match b2s_plicp_scan_match; /* opaque: B ScanMatchPLICP nodes */

/* One laser per recording: n_beams[b], angle_min[b], angle_increment[b] (the LaserScans' float32 fields).
 * B2S_ERR_BAD_PARAMS for NULL pointers, batch < 1, a beam count < 3 or icp.max_iterations < 1; B2S_ERR_NO_DEVICE
 * without a device; B2S_ERR_TOO_LARGE when a beam count is above the pair kernel's limit (2408 on an H100, 82 bytes of
 * shared memory per beam). */
b2s_status b2s_plicp_scan_match_create(const b2s_icp_params *params, int batch, const int32_t *n_beams,
                                       const float *angle_min, const float *angle_increment, int device,
                                       void *cuda_stream, b2s_plicp_scan_match **out);
void b2s_plicp_scan_match_destroy(b2s_plicp_scan_match *h);
/* ScanCallback on every recording's next n_scans[b] LaserScans (0: recording b is untouched), in ONE launch.
 * Recordings are processor-major and ragged: ranges holds n_scans[0] scans of n_beams[0] floats, then n_scans[1] scans
 * of n_beams[1] floats, ...; range_limits [sum n_scans][2] = each scan's (range_min, range_max); out [sum n_scans].
 * The handle keeps each recording's last scan and its range fields in device memory, so two calls over consecutive
 * parts of every recording equal one call.  B2S_ERR_BAD_PARAMS (nothing enqueued, nothing written) for NULL arrays or
 * a negative count. */
b2s_status b2s_plicp_scan_match_process(b2s_plicp_scan_match *h, const int32_t *n_scans, const float *ranges,
                                        const float *range_limits, b2s_plicp_scan_match_step *out);
/* a fresh node for one recording, or for all with recording = -1: its next scan initialises it */
b2s_status b2s_plicp_scan_match_reset(b2s_plicp_scan_match *h, int recording);

/* ---------------------------------------------------------------- lesson2: PCL ICP scan matching
 * ScanMatchICP (lesson2/src/scan_match_icp.cc): every LaserScan becomes a pcl::PointCloud<PointXYZ>
 * (ConvertScan2PointCloud, :89-130) and the previous cloud is aligned to the current one by a default-constructed
 * pcl::IterativeClosestPoint<PointXYZ, PointXYZ> (ScanMatchWithICP, :135-164).  align() gets no initial guess, so the
 * pairs of a recording are independent and a whole recording is one batch.  PARITY UNPINNED: PCL is third-party code
 * absent from the reference tree; its published behaviour (PCL 1.8) is restated, see DESIGN.md §2 and §4. */
/* The node default-constructs its ICP (scan_match_icp.h:49) and sets nothing on it (scan_match_icp.cc:137-143), so
 * every default below is PCL's own (parity unpinned). */
typedef struct b2s_pcl_icp_params {
  int32_t max_iterations;             /* max_iterations_, node default 10 (scan_match_icp.cc:143; parity unpinned).
                                         Reaching it counts as converged (failure_after_max_iter_ = false) */
  int32_t drop_invalid_points;        /* 0 = the node (scan_match_icp.cc:96-123; parity unpinned): a non-finite reading
                                         or one outside (range_min, range_max) stays in the cloud as a point at
                                         (0, 0, 0) and takes part in ICP.  1 = leave such readings out of both clouds */
  double max_correspondence_distance; /* corr_dist_threshold_, node default sqrt(DBL_MAX) = unlimited
                                         (scan_match_icp.cc:143; parity unpinned) */
  double transformation_epsilon;      /* transformation_epsilon_, node default 0 (scan_match_icp.cc:143; parity
                                         unpinned).  The rotation threshold is 1 - transformation_epsilon on cos(angle) */
  double euclidean_fitness_epsilon;   /* euclidean_fitness_epsilon_, node default -DBL_MAX = off
                                         (scan_match_icp.cc:143; parity unpinned) */
} b2s_pcl_icp_params;

typedef struct b2s_pcl_icp_result {
  float x[3];                /* getFinalTransformation() as (x, y, yaw), yaw = atan2(R10, R00)
                                (pcl::getTranslationAndEulerAngles, scan_match_icp.cc:156-161; parity unpinned).  It maps
                                the source (previous) scan into the target (current) scan's frame.  When an odd number
                                of the iterations fitted a reflection (PCL's 3-D SVD fit of planar points takes the
                                in-plane mirror with z -> -z where the cross-covariance has a negative determinant), the
                                2x2 block is a reflection [[c, s], [s, -c]]: it is reported the same way, yaw =
                                atan2(s, c), and the mirror itself is not reported */
  int32_t converged;         /* hasConverged() (scan_match_icp.cc:148; parity unpinned) */
  int32_t iterations;        /* iterations run, nr_iterations_ (scan_match_icp.cc:143; parity unpinned) */
  int32_t n_correspondences; /* correspondences of the last iteration (scan_match_icp.cc:143; parity unpinned) */
  double fitness_score;      /* getFitnessScore() (scan_match_icp.cc:145; parity unpinned): mean squared nearest-target
                                distance of the aligned source, DBL_MAX when no point has a target */
} b2s_pcl_icp_result;

/* ConvertScan2PointCloud + ScanMatchWithICP for `n_pairs` scan pairs on the device.  ranges [n_scans][n] (host) share
 * the LaserScan fields angle_min, angle_increment, range_min, range_max (beam angle angle_min + i * angle_increment in
 * float, :112).  pairs [n_pairs][2] = (source, target) scan indices; NULL = the node's loop, (i - 1, i) for every i >= 1,
 * with n_pairs = n_scans - 1.  guesses [n_pairs][3] = (x, y, yaw) initial transforms, NULL = identity as the node
 * calls align().  Each scan is converted once, however many pairs use it.  B2S_ERR_TOO_LARGE when the beam count
 * does not fit the kernel's shared memory (32 bytes per beam). */
b2s_status b2s_pcl_icp_align(const b2s_pcl_icp_params *params, int n_scans, int n, const float *ranges, float angle_min,
                             float angle_increment, float range_min, float range_max, int n_pairs, const int32_t *pairs,
                             const float *guesses, int device, void *cuda_stream, b2s_pcl_icp_result *results);

/* ---------------------------------------------------------------- lesson5: motion de-skew pre-stage (SURVEY.md §8(f).4)
 * LidarUndistortion (lesson5/src/lidar_undistortion.cc): every reading of a LaserScan is moved into the sensor frame
 * of the scan's first valid reading, using IMU angles integrated over the scan and the odometry increment across it.
 * The per-beam loop (CorrectLaserScan, :339-393) runs on the device for a batch of scans; the per-scan preparation is
 * host arithmetic.  Pinned to the unmodified node (tests/test_deskew_reference.py, tests/test_gpu_deskew_edges.py)
 * except pcl::getTransformation and Eigen::Affine3f inverse / product: those are third-party header code absent from
 * the reference tree (PCL 1.8, Eigen 3.3), and their published algorithms are restated. */
typedef struct b2s_deskew_scan {
  double time_start, time_increment;   /* header.stamp (start of the sweep), LaserScan::time_increment */
  float range_min, range_max;          /* readings outside [range_min, range_max] or non-finite are skipped (:349-352) */
  int32_t use_imu, use_odom;           /* the node's use_imu_ / use_odom_ */
  int32_t imu_last, reserved;          /* current_imu_index_ after PruneImuDeque: index of the last table entry */
  double odom_start_time, odom_end_time; /* stamps of start_odom_msg_ / end_odom_msg_ */
  float odom_incre[3];                 /* odom_incre_x_/y_/z_ */
  float reserved2;
} b2s_deskew_scan;

/* PruneImuDeque's integration (:196-238) over the IMU messages of the (already pruned) queue: stamp[n_imu],
 * angular_velocity[n_imu][3]; fills imu_time / rot_x / rot_y / rot_z [capacity] (zeroed first, as ResetParameters does)
 * and returns current_imu_index_ (the last entry), or -2 where the node would run outside its arrays. */
int32_t b2s_deskew_integrate_imu(int n_imu, const double *stamp, const double *angular_velocity, double scan_time_start,
                                 double scan_time_end, int capacity, double *imu_time, double *rot_x, double *rot_y,
                                 double *rot_z);
/* PruneOdomDeque's increment (:296-333): start / end pose as (x, y, z, roll, pitch, yaw) — the position of the
 * odometry message and tf::Matrix3x3(orientation).getRPY — gives odom_incre_x_/y_/z_. */
void b2s_deskew_odom_increment(const double start_pose[6], const double end_pose[6], float out_increment[3]);
/* CorrectLaserScan for `batch` scans (any batch >= 1; n_beams <= 65535 * 256): ranges [batch][n_beams] (host),
 * per-scan parameters, IMU tables [batch][imu_stride]; out_xyz [batch][n_beams][3] (host): the corrected point cloud,
 * skipped readings as (0, 0, 0) (the cloud is cleared and resized per scan).  angle_min and angle_increment are the
 * LaserScan's float32 fields: they are rounded to float and beam i's angle is summed in float, angle_min + i *
 * angle_increment, as CreateAngleCache (:162-174) sums them, before its cos / sin are taken in double. */
b2s_status b2s_lidar_undistort(int batch, int n_beams, const float *ranges, double angle_min, double angle_increment,
                               const b2s_deskew_scan *scans, const double *imu_time, const double *imu_rot_x,
                               const double *imu_rot_y, const double *imu_rot_z, int imu_stride, float *out_xyz, int device,
                               void *cuda_stream);

/* The whole node over one recording of one laser: LidarUndistortion's callbacks (:82-159) and queue pruning
 * (PruneImuDeque :177-249, PruneOdomDeque :252-336) on the host, CorrectLaserScan for every published scan on the
 * device.  The node's AsyncSpinner serves the three streams under separate locks, so what it saw at a scan's callback
 * is the number of IMU and odometry messages delivered before it: imu_arrived / odom_arrived, non-decreasing over the
 * scans.  Scan k is corrected at the callback of scan k + 1 with the messages delivered by then, so the last scan is
 * never published; a scan whose queues do not cover it is dropped.  The angle cache and the beam count come from the
 * first scan, as the node caches them; stamp, time_increment, range_min and range_max from each.  Stamps are
 * (sec, nsec) and compared as ros::Time::toSec doubles.  tf's quaternionMsgToTF and Matrix3x3::getRPY are restated on the
 * host (a zero quaternion, the default of a message the node never received, gives NaN angles). */
typedef struct b2s_imu_msg {
  uint32_t sec, nsec;
  double angular_velocity[3];
} b2s_imu_msg;
typedef struct b2s_odom_msg {
  uint32_t sec, nsec;
  double position[3], orientation[4]; /* quaternion x, y, z, w */
} b2s_odom_msg;
typedef struct b2s_deskew_node_scan {
  uint32_t sec, nsec;                   /* header.stamp */
  float time_increment, range_min, range_max;
  int32_t imu_arrived, odom_arrived;    /* messages of each log delivered before this scan's callback */
  int32_t reserved;                     /* 0 */
} b2s_deskew_node_scan;

/* out_status values, per corrected scan */
#define B2S_DESKEW_PUBLISHED 0  /* the node published the scan's cloud */
#define B2S_DESKEW_HELD 1       /* the recording's last scan: still in the laser queue */
#define B2S_DESKEW_WAIT_IMU 2   /* "Waiting for IMU data": the IMU queue is empty or does not cover the scan */
#define B2S_DESKEW_IMU_EMPTY 3  /* the IMU queue was pruned empty */
#define B2S_DESKEW_WAIT_ODOM 4  /* "Waiting for Odometry data" */
#define B2S_DESKEW_ODOM_EMPTY 5 /* the odometry queue was pruned empty */
#define B2S_DESKEW_UNDEFINED 6  /* the node's IMU integration reads imu_time_[-1] (the first message it integrates is
                                   at or after the scan start) or passes its 2000-entry table */

/* ranges [n_scans][n_beams] (host); imu [n_imu] and odom [n_odom] in delivery order (NULL allowed where the flag is off
 * or the count is 0).  out_status [n_scans]: a B2S_DESKEW_* value per scan.  out_state [n_scans] (may be NULL): the
 * b2s_deskew_scan a published row was computed from (imu_last -1 where an IMU gap covers the whole scan: the node then
 * takes rotation 0 throughout), or an undefined row's with imu_last -2; other rows are zero bytes.  Fed with the IMU
 * table b2s_deskew_integrate_imu returns over the pruned queue, it reproduces the row through b2s_lidar_undistort.
 * out_xyz [n_scans][n_beams][3] (host): the published cloud, zero bytes in every other row.  Refused before anything is
 * written: B2S_ERR_BAD_PARAMS for NULL arrays, negative counts, n_beams < 1, arrival counts that decrease or exceed
 * their log, or a NULL log whose flag is on.  n_scans == 0 does nothing and needs no device; otherwise
 * B2S_ERR_NO_DEVICE without one.  The odometry prune still runs after an undefined IMU integration, as the node goes
 * on; an undefined row keeps that status whatever the odometry prune finds.  Returns when the clouds are on the host. */
b2s_status b2s_lidar_undistortion_node(int use_imu, int use_odom, float angle_min, float angle_increment, int n_beams,
                                       int n_scans, const b2s_deskew_node_scan *scans, const float *ranges, int n_imu,
                                       const b2s_imu_msg *imu, int n_odom, const b2s_odom_msg *odom, int32_t *out_status,
                                       b2s_deskew_scan *out_state, float *out_xyz, int device, void *cuda_stream);

/* B LidarUndistortion nodes behind one handle, one laser per recording, fed in parts: each call hands every recording
 * its next LaserScans and the IMU and odometry messages delivered with them, and the handle keeps each node's state
 * across calls.  All recordings' published scans run in ONE launch (one CTA per scan, grid x up to 2^31 - 1).
 * b2s_lidar_undistortion_node is this handle's path for one fresh recording, its rows shifted to the corrected scan. */
#define B2S_DESKEW_CACHED 7     /* handle rows only: the callback of the node's first scan (ever or since reset) only
                                   cached that scan */

typedef struct b2s_deskew_node b2s_deskew_node; /* opaque: B LidarUndistortion nodes */
typedef struct b2s_deskew_laser {               /* what the node takes from its first scan */
  float angle_min, angle_increment;             /* CreateAngleCache's float fields */
  int32_t n_beams;                              /* scan_count_ */
  int32_t use_imu, use_odom;                    /* use_imu_ / use_odom_ */
  int32_t reserved;                             /* 0 */
} b2s_deskew_laser;

/* lasers [batch].  B2S_ERR_BAD_PARAMS, before the device is touched, for batch < 1, n_beams < 1 or NULL pointers;
 * B2S_ERR_NO_DEVICE without a device.  cuda_stream NULL: the handle makes its own. */
b2s_status b2s_deskew_node_create(int batch, const b2s_deskew_laser *lasers, int device, void *cuda_stream,
                                  b2s_deskew_node **out);
void b2s_deskew_node_destroy(b2s_deskew_node *h);
/* a fresh node for one recording, or for all with recording = -1: its next scan is cached as the first.
 * B2S_ERR_BAD_PARAMS for a recording outside [-1, batch). */
b2s_status b2s_deskew_node_reset(b2s_deskew_node *h, int recording);
/* The callbacks of every recording's next n_scans[b] LaserScans (0 leaves recording b's scans as they are; its new
 * messages still join its queues).
 *
 * Layout: arrays are recording-major and ragged.  scans, out_status and out_state have sum n_scans rows.  ranges holds
 * n_scans[0] rows of n_beams[0] floats, then n_scans[1] rows of n_beams[1] floats, and so on; out_xyz has the same
 * shape with 3 floats per beam.  imu has sum n_imu messages and odom sum n_odom, each recording's in delivery order.
 *
 * Arrival counts: a scan's imu_arrived / odom_arrived count its recording's messages OF THIS CALL delivered before its
 * callback; they do not decrease and do not exceed that recording's count.  Messages after the last scan's count are
 * delivered before the next call's first scan.  Messages of a recording whose flag is off are ignored.
 *
 * Rows are callback-indexed: row k of a recording in a call is what the callback of that call's k-th scan did.  It
 * corrected the scan handed in just before it (for k = 0, the previous call's last scan), with the statuses, states
 * and clouds of b2s_lidar_undistortion_node; or, for the node's first scan ever or since reset, it only cached the
 * scan: B2S_DESKEW_CACHED, with zero state and cloud bytes.  B2S_DESKEW_HELD is never returned: the held scan stays in
 * the handle.  Over a whole recording, rows 1 .. S - 1 therefore equal b2s_lidar_undistortion_node's rows 0 .. S - 2
 * byte for byte, however the recording is cut into calls.  out_state may be NULL.
 *
 * State kept per recording: the first-scan flag; the held scan's stamp and float fields, its ranges on the device; the
 * IMU and odometry queues, as copies of the messages not yet pruned (they grow as the node's deques do while a scan
 * waits); start_odom_msg_ and end_odom_msg_.
 *
 * B2S_ERR_BAD_PARAMS, before anything is enqueued or written and with every recording's state unchanged, for NULL
 * arrays where a count is non-zero (n_scans, n_imu and n_odom are always needed), negative counts, arrival counts that
 * decrease or exceed their log, or a NULL log whose flag is on for some recording.  A device error marks the handle
 * failed: later calls answer B2S_ERR_BAD_STATE.  Returns when the clouds are on the host. */
b2s_status b2s_deskew_node_process(b2s_deskew_node *h, const int32_t *n_scans, const b2s_deskew_node_scan *scans,
                                   const float *ranges, const int32_t *n_imu, const b2s_imu_msg *imu, const int32_t *n_odom,
                                   const b2s_odom_msg *odom, int32_t *out_status, b2s_deskew_scan *out_state,
                                   float *out_xyz);

/* ---------------------------------------------------------------- lesson1: corner-feature extraction
 * LaserScan::ScanCallback (lesson1/src/feature_detection.cc:77-179): the finite readings of a scan, a curvature
 * c = d * d from an 11-reading stencil (:112-124), and in each of six sectors the first 20 entries above edge_threshold
 * walked down a std::sort-ed range (:139-171).  Bit-identical to the node, ties included: where the 20th pick is tied
 * the device sorts that sector with a restatement of libstdc++'s introsort.  Every call is stateless. */
#define B2S_FEATURE_MAX_BEAMS 1500 /* max_scan_count (feature_detection.cc:23) */

/* ranges [batch][n] (host) -> out_ranges [batch][n] (host): the first n entries of the published corner_scan.ranges,
 * a picked beam's range and 0 elsewhere (the node's entries n .. 1499 are always 0; a picked range of 0 is invisible).
 * out_count [batch] (may be NULL): the number of picks, or -1 for a scan with a NaN curvature (finite ranges of
 * magnitude around 1e37 overflow the stencil both ways; the node's std::sort is undefined on it), whose out_ranges row
 * is all 0.  out_curvature [batch][n] (may be NULL): c at the beam of each reading the stencil covers, NaN at every
 * other beam; every NaN in it is the quiet NaN 0x7fc00000.  edge_threshold is the node's edge_threshold_ (1.0, :69).  B2S_ERR_BAD_PARAMS for a NULL ranges or
 * out_ranges, batch < 0, n < 0, or a negative or NaN edge_threshold (which would pick the node's {0, 0} placeholders);
 * B2S_ERR_TOO_LARGE for n > B2S_FEATURE_MAX_BEAMS, where the node overflows its buffer.  batch == 0 or n == 0 does
 * nothing, but still requires a device.  Returns when the results are on the host. */
b2s_status b2s_feature_detect(int batch, int n, const float *ranges, float edge_threshold, float *out_ranges,
                              int32_t *out_count, float *out_curvature, int device, void *cuda_stream);

/* ---------------------------------------------------------------- lesson4: the make-map nodes over whole recordings
 * lesson4's GMapping node (src/gmapping/gmapping.cc) and Hector make-map node (src/hector_mapping/hector_mapping.cc)
 * each build a fresh map from every LaserScan with the robot at the origin and publish it as a nav_msgs/OccupancyGrid.
 * These calls return, for every scan of a recording, the `data` payload the node publishes, bit for bit
 * (tests/test_lesson4_nodes_reference.py pins the restatement to the unmodified nodes, tests/test_gpu_lesson4_nodes.py
 * the device to the restatement).  One laser per call: `geometry` stands in for the node's first scan (angle_min,
 * angle_increment, range_min, range_max, n_ranges; its `ranges` pointer is not read).  ranges [n_scans][n_ranges]
 * float32 (host); out_maps [n_scans][height][width] int8 (host; page-locked memory lets the copies overlap the
 * compute), every byte defined.  out_dims = (width, height) as the node sizes its message; with out_maps NULL the call
 * only fills out_dims and needs no device.  Scans are independent: calls over consecutive chunks of a recording equal
 * one call.  n_scans == 0 does nothing.  Refused before anything is written: B2S_ERR_BAD_PARAMS for NULL arguments
 * (ranges may be NULL only when out_maps is NULL or n_scans is 0), negative counts or unusable bounds;
 * B2S_ERR_TOO_LARGE for n_ranges above B2S_NODE_MAPS_MAX_RANGES or a payload of 2^31 bytes or more.
 * The beams' unit vectors are taken on the host with the C library; no transcendental function runs on the device.
 * Returns when the maps are on the host. */
#define B2S_NODE_MAPS_MAX_RANGES 16384

typedef struct b2s_gmapping_node_params { /* GMapping::InitParams (gmapping.cc:44-84); node defaults in brackets */
  double max_range;     /* maxRange [30 - 0.01]: beams longer than this, 0 or non-finite are skipped */
  double max_use_range; /* maxUrange [25]: longer beams are clipped to it and mark no hit */
  double xmin, ymin, xmax, ymax; /* map bounds [-40, -40, 40, 40] */
  double delta;         /* cell size [0.05] */
  double occ_thresh;    /* occupied above this hit fraction [0.25] */
} b2s_gmapping_node_params;

/* GMapping::ScanCallback on every scan.  width = (xmax - xmin) / (float)delta truncated, as the node divides by the
 * message's float32 resolution (gmapping.cc:72-73): 1599 at the defaults, while the map's storage is 1600 x 1600
 * (ceil((xmax - xmin) / delta) rounded down to 32-cell patches, map.h:133).  Storage cell (x, y) is published at
 * MAP_IDX(width, x, y) = width * y + x, x outer and y inner, so a later cell overwrites an earlier one at the same byte
 * (at the defaults storage column 1599 of row y lands on byte (0, y + 1)); writes at or past width * height, where the
 * node overruns its own buffer (1 601 writes on 1 600 bytes at the defaults), are dropped; a byte no storage cell
 * reaches is 0, as the node's resized vector leaves it.  The beam cache is CreateCache's (:112-124): angle_min +
 * i * angle_increment summed in float, then the C library's double cos / sin.  B2S_ERR_OUT_OF_RANGE, with the first
 * such scan named in b2s_last_error(), when a kept beam's end cell or the laser's cell lies outside the storage (the
 * node's assert, map.h:186-191); nothing is written then.  B2S_ERR_BAD_PARAMS also when the storage is smaller than
 * one 32-cell patch. */
b2s_status b2s_gmapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_gmapping_node_params *params,
                                  int n_scans, const float *ranges, int32_t out_dims[2], int8_t *out_maps, int device,
                                  void *cuda_stream);

typedef struct b2s_hector_mapping_node_params { /* HectorMapping::InitParams (hector_mapping.cc:44-79) */
  double xmin, ymin, xmax, ymax; /* map bounds [-40, -40, 40, 40] */
  float delta;                   /* resolution_, a float in the node [0.05] */
  float reserved;                /* 0 */
} b2s_hector_mapping_node_params;

/* HectorMapping::ScanCallback on every scan.  width = (int)((xmax - xmin) / delta), height likewise (1599 x 1599 at
 * the defaults).  A beam is kept iff range_min < r < range_max - 0.1f (:150-156); its point is (cos(a) * r,
 * sin(a) * r) in double rounded to float, the angle a accumulated in float beam by beam (:144-163) and cos / sin the
 * C library's double functions, as the node's unqualified call on a float resolves where <math.h> is not included
 * (DESIGN §7).  updateByScanJustOnce (OccGridMapBase.h:175-217) draws every kept beam from cell (800, 800) to
 * (800, 800) + (int)round(p / 0.05), whatever delta is, when the two differ and both lie inside the map.  Each byte
 * is 100 where a drawn beam ends, else 0 where one passes, else -1 (PublishMap, :177-211). */
b2s_status b2s_hector_mapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_hector_mapping_node_params *params,
                                        int n_scans, const float *ranges, int32_t out_dims[2], int8_t *out_maps,
                                        int device, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SLAM_H */
