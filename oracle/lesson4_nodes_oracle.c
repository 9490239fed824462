/*
 * lesson4_nodes_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 * Plain-C restatement of lesson4's two make-map nodes over a recording, written around the restatements that are
 * already pinned (compiled into the same library by oracle/lesson4_nodes_port.py):
 *   GMapping node   src/gmapping/gmapping.cc:44-242 (InitParams sizing, CreateCache on the first scan, a fresh
 *                   ScanMatcherMap per scan, PublishMap) around gmapping_oracle.c's orc_gmap_compute_map / orc_gmap_ros
 *   Hector node     src/hector_mapping/hector_mapping.cc:44-211 (InitParams sizing, ROSLaserScanToDataContainer, a
 *                   fresh GridMap per scan, PublishMap) around hector_oracle.c's orc_hmap_update_by_scan_just_once
 * PINNED against the unmodified nodes (oracle/ref_lesson4_gmapping.cpp, oracle/ref_lesson4_hector.cpp ->
 * oracle/_ref/liblesson4_ref.so) by tests/test_lesson4_nodes_reference.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h"

/* gmapping_oracle.c */
void orc_gmap_layout(double cx, double cy, double xmin, double ymin, double xmax, double ymax, double delta,
                     int32_t out[4]);
int orc_gmap_compute_map(double cx, double cy, double delta, const int32_t layout[4], const double *ranges,
                         const double *angles, int nb, double laser_x, double laser_y, double max_range,
                         double max_use_range, int32_t *n, int32_t *visits, float *acc_x, float *acc_y);
void orc_gmap_ros(const int32_t layout[4], const int32_t *n, const int32_t *visits, double occ_thresh, int width,
                  int height, int8_t *out);
/* hector_oracle.c (its map type is opaque here) */
struct orc_hmap_opaque;
struct orc_hmap_opaque *orc_hmap_create(int size_x, int size_y, float resolution, float start_x, float start_y);
void orc_hmap_destroy(struct orc_hmap_opaque *m);
void orc_hmap_copy(const struct orc_hmap_opaque *m, float *log_odds, int32_t *update_index);
long orc_hmap_update_by_scan_just_once(struct orc_hmap_opaque *m, const float *points, int n, const float origo[2]);

/* the node's conversion of a double map dimension into its unsigned / int field; -1 where it is not a usable size */
static int node_dim(double d) { return d >= 1.0 && d < 2147483648.0 ? (int)d : -1; }

/* InitParams (gmapping.cc:69-73): map_.info.width / height = (max - min) / (float)resolution, truncated */
int orc_gmapping_node_dims(const b2s_gmapping_node_params *p, int32_t dims[2]) {
  dims[0] = node_dim((p->xmax - p->xmin) / (double)(float)p->delta);
  dims[1] = node_dim((p->ymax - p->ymin) / (double)(float)p->delta);
  return dims[0] > 0 && dims[1] > 0 ? 0 : -1;
}

/* ScanCallback on every scan of ranges [n_scans][geometry->n_ranges].  out_maps [n_scans][height][width]: the
 * published data.  overrun [n_scans][overrun_cap] (may be NULL): the bytes PublishMap writes at width*height + k,
 * 0x55 where it writes none; n_overrun [n_scans] (read with overrun): how many distinct such bytes it writes.  Returns the
 * index of the first scan whose rays leave the storage (the node asserts there; maps before it are filled), n_scans
 * when there is none, or -1 for bounds the node cannot size. */
int orc_gmapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_gmapping_node_params *p, int n_scans,
                           const float *ranges, int8_t *out_maps, int8_t *overrun, int overrun_cap, int32_t *n_overrun) {
  int32_t dims[2], L[4];
  if (orc_gmapping_node_dims(p, dims)) return -1;
  const int width = dims[0], height = dims[1], nb = geometry->n_ranges;
  const double cx = (p->xmin + p->xmax) / 2.0, cy = (p->ymin + p->ymax) / 2.0; /* PublishMap (:130-135) */
  orc_gmap_layout(cx, cy, p->xmin, p->ymin, p->xmax, p->ymax, p->delta, L);
  if (L[0] <= 0 || L[1] <= 0) return -1;
  const size_t cells = (size_t)L[0] * L[1], wh = (size_t)width * height;
  /* CreateCache (:112-124): the angle angle_min + i * angle_increment is a float sum, widened to double */
  double *angles = (double *)malloc(sizeof(double) * (nb > 0 ? nb : 1));
  double *d = (double *)malloc(sizeof(double) * (nb > 0 ? nb : 1));
  for (int i = 0; i < nb; i++) angles[i] = (double)(geometry->angle_min + (float)(unsigned)i * geometry->angle_increment);
  int32_t *n = (int32_t *)malloc(cells * 4), *visits = (int32_t *)malloc(cells * 4);
  float *ax = (float *)malloc(cells * 4), *ay = (float *)malloc(cells * 4);
  int first_bad = n_scans;
  for (int s = 0; s < n_scans && first_bad == n_scans; s++) {
    const float *r = ranges + (size_t)s * nb;
    int kept = 0;
    for (int i = 0; i < nb; i++) {
      d[i] = (double)r[i];
      kept |= !(d[i] > p->max_range || d[i] == 0.0 || !isfinite(d[i])); /* ComputeMap's filter (:190-191) */
    }
    memset(n, 0, cells * 4); memset(visits, 0, cells * 4);
    memset(ax, 0, cells * 4); memset(ay, 0, cells * 4);
    /* a kept beam whose cells leave the storage hits map.h's assert; with none kept, the laser's cell is never read */
    if (kept && orc_gmap_compute_map(cx, cy, p->delta, L, d, angles, nb, 0.0, 0.0, p->max_range, p->max_use_range, n,
                                     visits, ax, ay)) {
      first_bad = s;
      break;
    }
    orc_gmap_ros(L, n, visits, p->occ_thresh, width, height, out_maps + (size_t)s * wh);
    if (overrun) { /* the writes orc_gmap_ros drops: MAP_IDX(width, x, y) >= width * height */
      int8_t *ov = overrun + (size_t)s * overrun_cap;
      memset(ov, 0x55, (size_t)overrun_cap);
      int32_t count = 0;
      for (int x = 0; x < L[0]; x++)
        for (int y = 0; y < L[1]; y++) {
          const size_t o = (size_t)width * y + x, c = (size_t)x + (size_t)y * L[0];
          if (o < wh || o - wh >= (size_t)overrun_cap) continue;
          const double occ = visits[c] ? (double)n[c] * 1 / (double)visits[c] : -1;
          count += ov[o - wh] == 0x55;
          ov[o - wh] = occ < 0 ? -1 : (occ > p->occ_thresh ? 100 : 0);
        }
      if (n_overrun) n_overrun[s] = count;
    }
  }
  free(angles); free(d); free(n); free(visits); free(ax); free(ay);
  return first_bad;
}

/* InitParams (hector_mapping.cc:57-58): map_size_ = (max - min) / resolution_, resolution_ a float */
int orc_hector_mapping_node_dims(const b2s_hector_mapping_node_params *p, int32_t dims[2]) {
  dims[0] = node_dim((p->xmax - p->xmin) / (double)p->delta);
  dims[1] = node_dim((p->ymax - p->ymin) / (double)p->delta);
  return dims[0] > 0 && dims[1] > 0 ? 0 : -1;
}

/* ScanCallback on every scan: out_maps [n_scans][height][width].  Returns 0, or -1 for bounds the node cannot size. */
int orc_hector_mapping_node_maps(const b2s_laser_scan_msg *geometry, const b2s_hector_mapping_node_params *p,
                                 int n_scans, const float *ranges, int8_t *out_maps) {
  int32_t dims[2];
  if (orc_hector_mapping_node_dims(p, dims)) return -1;
  const int width = dims[0], height = dims[1], nb = geometry->n_ranges;
  const size_t wh = (size_t)width * height;
  float *pts = (float *)malloc(sizeof(float) * 2 * (nb > 0 ? nb : 1));
  float *lo = (float *)malloc(sizeof(float) * wh);
  const float max_range = geometry->range_max - 0.1f, origo[2] = {0.0f, 0.0f};
  for (int s = 0; s < n_scans; s++) {
    const float *r = ranges + (size_t)s * nb;
    /* ROSLaserScanToDataContainer (:138-165): the float angle accumulates; cos / sin resolve to the double functions */
    float angle = geometry->angle_min;
    int k = 0;
    for (int i = 0; i < nb; i++) {
      const float dist = r[i];
      if (dist > geometry->range_min && dist < max_range) {
        pts[2 * k] = (float)(cos((double)angle) * (double)dist);
        pts[2 * k + 1] = (float)(sin((double)angle) * (double)dist);
        k++;
      }
      angle += geometry->angle_increment;
    }
    struct orc_hmap_opaque *m = orc_hmap_create(width, height, p->delta, 0.0f, 0.0f); /* a new GridMap (:94) */
    orc_hmap_update_by_scan_just_once(m, pts, k, origo);
    orc_hmap_copy(m, lo, NULL);
    orc_hmap_destroy(m);
    /* PublishMap (:177-211): memset -1, then 0 where isFree (log-odds < 0), 100 where isOccupied (> 0) */
    int8_t *out = out_maps + (size_t)s * wh;
    memset(out, -1, wh);
    for (size_t i = 0; i < wh; i++) {
      if (lo[i] < 0.0f) out[i] = 0;
      else if (lo[i] > 0.0f) out[i] = 100;
    }
  }
  free(pts); free(lo);
  return 0;
}
