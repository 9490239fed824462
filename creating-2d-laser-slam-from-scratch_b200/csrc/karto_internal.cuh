// The Karto modules' internal interfaces (not part of the C ABI): the Mapper and its match pool (karto_mapper.cu), the
// batched occupancy-grid build (karto_occgrid.cu) and the LaserScan conversion (ros_io.cu), as the node batch
// (karto_node.cu) drives them.  Every file that defines or calls one of these includes this header.
#pragma once
#include <utility>
#include <vector>

#include "common.cuh"

namespace b2s {

// ---- karto_mapper.cu

// One batch of a Mapper's matches: base scans are named by their unique id in `mapper`, base_ids / base_poses
// [batch][max_base] padded by repeating a match's last base scan.
struct MatchRequest {
  const b2s_mapper *mapper = nullptr;
  int which = 0, batch = 0, max_base = 0, do_penalize = 0, do_refine = 0;
  const double *ranges = nullptr, *poses = nullptr, *base_poses = nullptr;
  const int32_t *base_ids = nullptr;
  b2s_match_result *results = nullptr;
};
// A Mapper made by mapper_create_fleet hands each batch to `FleetMatchFn`, which runs it on a MatchPool: the Mapper's
// own (b2s_mapper_create) or one shared by the nodes of a Karto node batch (karto_node.cu).
typedef b2s_status (*FleetMatchFn)(void *user, const MatchRequest &r);
b2s_status mapper_create_fleet(const b2s_mapper_params *params, const b2s_laser *laser, FleetMatchFn match, void *user,
                               b2s_mapper **out);
const double *mapper_scan_ranges(const b2s_mapper *m, int id);

struct MatchPool;
b2s_status match_pool_create(const b2s_matcher_params params[2], const b2s_laser &laser, int device, int clients,
                             int scan_buffer_size, MatchPool **out);
void match_pool_destroy(MatchPool *p);
b2s_status match_pool_serve(MatchPool *p, const std::vector<std::pair<int, const MatchRequest *>> &group, double *counts);

// ---- karto_occgrid.cu

struct OccBatch;
b2s_status occ_batch_create(const b2s_laser &laser, int device, OccBatch **out);
void occ_batch_destroy(OccBatch *b);
double occ_batch_bytes_d2h(const OccBatch *b);
b2s_status occ_batch_append(OccBatch *b, int count, const float *rows, int32_t *first);
b2s_status occ_batch_build(OccBatch *b, int G, const int32_t *n_scans, const int32_t *rows, const double *poses,
                           const double *resolution, b2s_occ_grid_info *info, int32_t *have, const int8_t **payload);

// ---- ros_io.cu

b2s_status karto_laser_from_msg(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                                b2s_laser *out);

}  // namespace b2s
