// TEST INFRASTRUCTURE — CSM's sm_params / sm_result / LDP as lesson3's plicp_odometry.cc uses them, with sm_icp answered
// by the PL-ICP restatement orc_plicp_match (oracle/plicp_oracle.c), for compiling the node unmodified
// (oracle/ref_lesson3.cpp).  CSM itself is an external, un-versioned dependency (PARITY UNPINNED, DESIGN.md §7).
//
// The node's values of the switches the restatement does not model have no effect on the result: use_corr_tricks only
// speeds up the correspondence search, and restart, do_alpha_test, do_visibility_test, do_compute_covariance,
// use_ml_weights, use_sigma_weights and debug_verify_tricks are 0.  sm_icp refuses (throws) any other value of those
// switches rather than ignore it; sigma, clustering_threshold, orientation_neighbourhood and the restart thresholds only
// matter under the switches above or for the covariance.
#pragma once

#include <cmath>
#include <cstdlib>
#include <stdexcept>

#include "../../../include/b200slam.h"

extern "C" int orc_plicp_match(const b2s_icp_params *P, int n, const double *ref_r, const double *sens_r,
                               const double *theta, double range_min, double range_max, const double first_guess[3],
                               b2s_icp_result *out);

struct gsl_matrix {};
inline void gsl_matrix_free(gsl_matrix *m) { delete m; }

struct laser_data {
  int nrays = 0;
  double min_theta = 0, max_theta = 0;
  double *theta = nullptr, *readings = nullptr;
  int *valid = nullptr, *cluster = nullptr;
  double odometry[3] = {0, 0, 0}, estimate[3] = {0, 0, 0}, true_pose[3] = {0, 0, 0};
};
typedef laser_data *LDP;

inline LDP ld_alloc_new(int n) {
  LDP l = new laser_data();
  l->nrays = n;
  l->theta = new double[n];
  l->readings = new double[n];
  l->valid = new int[n];
  l->cluster = new int[n];
  return l;
}
inline void ld_free(LDP l) {
  if (!l) return;
  delete[] l->theta;
  delete[] l->readings;
  delete[] l->valid;
  delete[] l->cluster;
  delete l;
}

struct sm_params {
  LDP laser_ref = nullptr, laser_sens = nullptr;
  double first_guess[3] = {0, 0, 0};
  double max_angular_correction_deg = 0, max_linear_correction = 0;
  int max_iterations = 0;
  double epsilon_xy = 0, epsilon_theta = 0, max_correspondence_dist = 0, sigma = 0;
  int use_corr_tricks = 0, restart = 0;
  double restart_threshold_mean_error = 0, restart_dt = 0, restart_dtheta = 0, clustering_threshold = 0;
  int orientation_neighbourhood = 0, use_point_to_line_distance = 0, do_alpha_test = 0;
  double do_alpha_test_thresholdDeg = 0, outliers_maxPerc = 0, outliers_adaptive_order = 0, outliers_adaptive_mult = 0;
  int do_visibility_test = 0, outliers_remove_doubles = 0, do_compute_covariance = 0, debug_verify_tricks = 0;
  int use_ml_weights = 0, use_sigma_weights = 0;
  double laser[3] = {0, 0, 0};
  double min_reading = 0, max_reading = 0;
};

struct sm_result {
  int valid = 0;
  double x[3] = {0, 0, 0};
  int iterations = 0, nvalid = 0;
  double error = 0;
  gsl_matrix *cov_x_m = nullptr, *dx_dy1_m = nullptr, *dx_dy2_m = nullptr;
};

inline void sm_icp(sm_params *in, sm_result *out) {
  if (in->restart || in->do_alpha_test || in->do_visibility_test || in->do_compute_covariance || in->use_ml_weights ||
      in->use_sigma_weights || in->debug_verify_tricks)
    throw std::runtime_error("sm_icp stand-in: a CSM switch the restatement does not model is set");
  const LDP r = in->laser_ref, s = in->laser_sens;
  const int n = r->nrays;
  if (s->nrays != n) throw std::runtime_error("sm_icp stand-in: scans of different lengths");
  double *rr = new double[n], *sr = new double[n];
  for (int i = 0; i < n; i++) {
    // the LDP's valid flags decide; an invalid reading goes in as NaN, which no range window accepts
    rr[i] = r->valid[i] ? r->readings[i] : NAN;
    sr[i] = s->valid[i] ? s->readings[i] : NAN;
  }
  b2s_icp_params p;
  p.max_angular_correction_deg = in->max_angular_correction_deg;
  p.max_linear_correction = in->max_linear_correction;
  p.epsilon_xy = in->epsilon_xy;
  p.epsilon_theta = in->epsilon_theta;
  p.max_correspondence_dist = in->max_correspondence_dist;
  p.outliers_maxPerc = in->outliers_maxPerc;
  p.outliers_adaptive_order = in->outliers_adaptive_order;
  p.outliers_adaptive_mult = in->outliers_adaptive_mult;
  p.max_iterations = in->max_iterations;
  p.use_point_to_line_distance = in->use_point_to_line_distance;
  p.outliers_remove_doubles = in->outliers_remove_doubles;
  p.reserved = 0;
  b2s_icp_result res;
  orc_plicp_match(&p, n, rr, sr, r->theta, -INFINITY, INFINITY, in->first_guess, &res);
  delete[] rr;
  delete[] sr;
  out->valid = res.valid;
  for (int k = 0; k < 3; k++) out->x[k] = res.x[k];
  out->iterations = res.iterations;
  out->nvalid = res.nvalid;
  out->error = res.error;
}
