/*
 * plicp_scan_match_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of lesson3's scan-to-scan node, ScanMatchPLICP (reference/lesson3/src/scan_match_plicp.cc:162-300):
 * the node's loop in C around the PL-ICP restatement orc_plicp_match (oracle/plicp_oracle.c).  Built with it into a
 * library of its own (oracle/plicp_scan_match_port.py), built by oracle/recipes.py.  The unmodified node,
 * compiled against the stand-ins under oracle/shim/ (oracle/ref_lesson3_scan_match.cpp), pins it bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

int orc_plicp_match(const b2s_icp_params *P, int n, const double *ref_r, const double *sens_r, const double *theta,
                    double range_min, double range_max, const double first_guess[3], b2s_icp_result *out);

/* LaserScanToLDP (:220-261) into the readings orc_plicp_match takes: double r valid iff range_min < r < range_max with
 * the message's own float fields; an invalid reading goes in as NaN, which the (-inf, inf) window of the call rejects,
 * so each scan keeps its own validity whatever the other scan's range fields are */
static void to_readings(const float *r, int n, float range_min, float range_max, double *out) {
  for (int i = 0; i < n; i++) {
    const double v = r[i];
    out[i] = (v > range_min && v < range_max) ? v : NAN;
  }
}

/* The node's loop for ONE recording from a fresh node: ranges [n_scans][n] float32, limits [n_scans][2] (range_min,
 * range_max of each scan) -> out [n_scans] as b2s_plicp_scan_match_process fills it */
void orc_plicp_scan_match(const b2s_icp_params *P, int n, float angle_min, float angle_increment, int n_scans,
                          const float *ranges, const float *limits, b2s_plicp_scan_match_step *out) {
  double *theta = malloc(sizeof(double) * n), *prev = malloc(sizeof(double) * n), *cur = malloc(sizeof(double) * n);
  for (int i = 0; i < n; i++) theta[i] = (double)(angle_min + (float)i * angle_increment); /* :243 */
  const double zero[3] = {0.0, 0.0, 0.0};
  for (int s = 0; s < n_scans; s++) {
    b2s_plicp_scan_match_step *o = out + s;
    memset(o, 0, sizeof *o);
    to_readings(ranges + (size_t)s * n, n, limits[2 * s], limits[2 * s + 1], cur);
    if (s > 0) {
      orc_plicp_match(P, n, prev, cur, theta, -INFINITY, INFINITY, zero, &o->icp); /* :275-284 */
      o->theta_deg = o->icp.x[2] * 180 / M_PI;                                    /* :289 */
      o->matched = 1;
    }
    double *t = prev; prev = cur; cur = t; /* :297-298 */
  }
  free(theta); free(prev); free(cur);
}
