/*
 * plicp_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the lesson3 fine-align stage: PL-ICP (point-to-line ICP) as the reference calls it,
 *   reference/lesson3/src/plicp_odometry.cc:285-322 (LaserScanToLDP), :391 (sm_icp), :72-185 (sm_params).
 *
 * PARITY UNPINNED.  The arithmetic lives in CSM (Andrea Censi's C Scan Matcher), pulled by the reference as the
 * system package `ros-kinetic-csm` (install_dependence.sh:4) with NO pinned version and absent from the reference checkout
 * and from this image; no reference test pins sm_icp's output.  This file restates the PUBLISHED algorithm
 * (A. Censi, "An ICP variant using a point-to-line metric", ICRA 2008) with the control flow of CSM's icp loop as
 * documented by its parameters (the subset the reference sets): per iteration
 *   1. transform the current scan with the running estimate,
 *   2. correspondences: nearest valid reference point j1 inside the angular window
 *      |dtheta| <= max_angular_correction + atan(max_linear_correction / |p|), within max_correspondence_dist, and its
 *      nearer valid index-neighbour j2 (the segment); extremal j1 are rejected (use_corr_tricks only accelerates this),
 *   3. outliers_remove_doubles: of all points mapped to the same j1 keep those within 3x the best squared distance,
 *   4. trimming: drop correspondences whose point-to-segment distance exceeds
 *      min(d[floor(n*outliers_maxPerc)], outliers_adaptive_mult * d[floor(n*outliers_adaptive_order)]),
 *   5. closed-form point-to-line solution (GPC: quadratic cost in (t, cos, sin), unit-norm constraint by a Lagrange
 *      multiplier = largest real root of a quartic),
 *   6. stop when the increment is below (epsilon_xy, epsilon_theta) or after max_iterations.
 * Acceptance: every iteration agrees with an independent float64 statement of the algorithm
 * (tests/plicp_reference.py) wherever no decision is within rounding of flipping, and known synthetic transforms are
 * recovered (tests/test_plicp.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h"

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

static int next_valid_up(const uint8_t *valid, int n, int j) {
  for (int k = j + 1; k < n; k++) if (valid[k]) return k;
  return -1;
}
static int next_valid_down(const uint8_t *valid, int j) {
  for (int k = j - 1; k >= 0; k--) if (valid[k]) return k;
  return -1;
}

static double dist_to_segment(const double a[2], const double b[2], const double x[2]) {
  double dx = b[0] - a[0], dy = b[1] - a[1];
  double len2 = dx * dx + dy * dy;
  double t = len2 > 0 ? ((x[0] - a[0]) * dx + (x[1] - a[1]) * dy) / len2 : 0.0;
  if (t < 0) t = 0;
  if (t > 1) t = 1;
  double px = a[0] + t * dx - x[0], py = a[1] + t * dy - x[1];
  return sqrt(px * px + py * py);
}

static int cmp_double(const void *a, const void *b) {
  double x = *(const double *)a, y = *(const double *)b;
  return (x > y) - (x < y);
}

/* largest real root of the monic quartic l^4 + c3 l^3 + c2 l^2 + c1 l + c0 (Durand-Kerner, fixed 200 sweeps) */
static double quartic_largest_real_root(double c3, double c2, double c1, double c0) {
  double re[4] = {1.0, 0.4, -0.65, 0.0}, im[4] = {0.0, 0.9, 0.72, -0.85};
  double scale = 1.0 + fmax(fmax(fabs(c3), fabs(c2)), fmax(fabs(c1), fabs(c0)));
  for (int k = 0; k < 4; k++) { re[k] *= scale; im[k] *= scale; }
  for (int it = 0; it < 200; it++) {
    for (int k = 0; k < 4; k++) {
      /* p(z) by Horner */
      double pr = 1.0, pi = 0.0, coef[4] = {c3, c2, c1, c0};
      for (int q = 0; q < 4; q++) {
        double nr = pr * re[k] - pi * im[k] + coef[q], ni = pr * im[k] + pi * re[k];
        pr = nr; pi = ni;
      }
      double dr = 1.0, di = 0.0;
      for (int j = 0; j < 4; j++) {
        if (j == k) continue;
        double ar = re[k] - re[j], ai = im[k] - im[j];
        double nr = dr * ar - di * ai, ni = dr * ai + di * ar;
        dr = nr; di = ni;
      }
      double den = dr * dr + di * di;
      if (den == 0.0) continue;
      re[k] -= (pr * dr + pi * di) / den;
      im[k] -= (pi * dr - pr * di) / den;
    }
  }
  double best = -1e300, tol = 1e-7 * scale;
  int found = 0;
  for (int k = 0; k < 4; k++)
    if (fabs(im[k]) <= tol && (!found || re[k] > best)) { best = re[k]; found = 1; }
  if (!found) { /* no real root numerically: take the root closest to the real axis */
    double bi = 1e300;
    for (int k = 0; k < 4; k++) if (fabs(im[k]) < bi) { bi = fabs(im[k]); best = re[k]; }
  }
  return best;
}

/* GPC: minimise sum (R p + t - q)^T C (R p + t - q) over (t, theta).  M = sum Mk^T C Mk (4x4 sym), g = -2 sum Mk^T C q */
static int gpc_solve(const double M[16], const double g[4], double x_out[3]) {
  double A[4] = {M[0], M[1], M[4], M[5]}, B[4] = {M[2], M[3], M[6], M[7]}, Dm[4] = {M[10], M[11], M[14], M[15]};
  double detA = A[0] * A[3] - A[1] * A[2];
  if (detA == 0.0) return 0;
  double Ai[4] = {A[3] / detA, -A[1] / detA, -A[2] / detA, A[0] / detA};
  /* AiB = A^-1 B ; S = D - B^T A^-1 B */
  double AiB[4] = {Ai[0] * B[0] + Ai[1] * B[2], Ai[0] * B[1] + Ai[1] * B[3], Ai[2] * B[0] + Ai[3] * B[2], Ai[2] * B[1] + Ai[3] * B[3]};
  double S[4] = {Dm[0] - (B[0] * AiB[0] + B[2] * AiB[2]), Dm[1] - (B[0] * AiB[1] + B[2] * AiB[3]),
                 Dm[2] - (B[1] * AiB[0] + B[3] * AiB[2]), Dm[3] - (B[1] * AiB[1] + B[3] * AiB[3])};
  double Sa[4] = {S[3], -S[1], -S[2], S[0]}; /* adj(S) */
  double p = S[0] + S[3], q = S[0] * S[3] - S[1] * S[2];
  /* v = (B^T A^-1 g1 - g2) / 2 */
  double Aig1[2] = {Ai[0] * g[0] + Ai[1] * g[1], Ai[2] * g[0] + Ai[3] * g[1]};
  double v[2] = {0.5 * ((B[0] * Aig1[0] + B[2] * Aig1[1]) - g[2]), 0.5 * ((B[1] * Aig1[0] + B[3] * Aig1[1]) - g[3])};
  double Sav[2] = {Sa[0] * v[0] + Sa[1] * v[1], Sa[2] * v[0] + Sa[3] * v[1]};
  double vv = v[0] * v[0] + v[1] * v[1], vSav = v[0] * Sav[0] + v[1] * Sav[1], vSa2v = Sav[0] * Sav[0] + Sav[1] * Sav[1];
  double lam = quartic_largest_real_root(2 * p, p * p + 2 * q - vv, 2 * p * q - 2 * vSav, q * q - vSa2v);
  double den = lam * lam + p * lam + q;
  if (den == 0.0) return 0;
  double r[2] = {(Sav[0] + lam * v[0]) / den, (Sav[1] + lam * v[1]) / den};
  double Br[2] = {B[0] * r[0] + B[1] * r[1] + 0.5 * g[0], B[2] * r[0] + B[3] * r[1] + 0.5 * g[1]};
  x_out[0] = -(Ai[0] * Br[0] + Ai[1] * Br[1]);
  x_out[1] = -(Ai[2] * Br[0] + Ai[3] * Br[1]);
  x_out[2] = atan2(r[1], r[0]);
  return isfinite(x_out[0]) && isfinite(x_out[1]) && isfinite(x_out[2]);
}

/* One scan pair.  ref/sens: n readings each on the beam angles theta[n]; valid iff range_min < r < range_max
 * (plicp_odometry.cc:291-301).  x: first guess in, estimate out (pose of sens in the ref frame). */
int orc_plicp_match(const b2s_icp_params *P, int n, const double *ref_r, const double *sens_r, const double *theta,
                    double range_min, double range_max, const double first_guess[3], b2s_icp_result *out) {
  double *rx = malloc(sizeof(double) * n), *ry = malloc(sizeof(double) * n);
  double *sx = malloc(sizeof(double) * n), *sy = malloc(sizeof(double) * n);
  double *wx = malloc(sizeof(double) * n), *wy = malloc(sizeof(double) * n);
  uint8_t *rv = malloc(n), *sv = malloc(n);
  int *j1 = malloc(sizeof(int) * n), *j2 = malloc(sizeof(int) * n);
  double *d2 = malloc(sizeof(double) * n), *dj = malloc(sizeof(double) * n), *ds = malloc(sizeof(double) * n), *sorted = malloc(sizeof(double) * n);
  for (int i = 0; i < n; i++) {
    rv[i] = ref_r[i] > range_min && ref_r[i] < range_max;
    sv[i] = sens_r[i] > range_min && sens_r[i] < range_max;
    rx[i] = rv[i] ? ref_r[i] * cos(theta[i]) : 0; ry[i] = rv[i] ? ref_r[i] * sin(theta[i]) : 0;
    sx[i] = sv[i] ? sens_r[i] * cos(theta[i]) : 0; sy[i] = sv[i] ? sens_r[i] * sin(theta[i]) : 0;
  }
  double x_old[3] = {first_guess[0], first_guess[1], first_guess[2]}, x_new[3] = {x_old[0], x_old[1], x_old[2]};
  const double min_theta = theta[0], max_theta = theta[n - 1];
  const double ang_res = (max_theta - min_theta) / n;
  const double max_d2 = P->max_correspondence_dist * P->max_correspondence_dist;
  int ok = 1, it = 0, nvalid = 0;
  double error = 0;
  for (it = 0; it < P->max_iterations; it++) {
    const double c = cos(x_old[2]), s = sin(x_old[2]);
    for (int i = 0; i < n; i++) {
      wx[i] = c * sx[i] - s * sy[i] + x_old[0];
      wy[i] = s * sx[i] + c * sy[i] + x_old[1];
      j1[i] = -1; j2[i] = -1;
      if (!sv[i]) continue;
      const double nrm = sqrt(wx[i] * wx[i] + wy[i] * wy[i]);
      const double delta = fabs(P->max_angular_correction_deg * M_PI / 180.0) + fabs(atan(P->max_linear_correction / nrm));
      const int range = (int)ceil(delta / ang_res);
      double st = atan2(wy[i], wx[i]);
      if (st < min_theta) st += 2 * M_PI;
      if (st > max_theta) st -= 2 * M_PI;
      const double start_cell = (st - min_theta) / (max_theta - min_theta) * n;
      int from = (int)floor(start_cell - range), to = (int)ceil(start_cell + range);
      if (from < 0) from = 0;
      if (from > n - 1) from = n - 1;
      if (to < 0) to = 0;
      if (to > n - 1) to = n - 1;
      int best = -1;
      double bd = 0;
      for (int j = from; j <= to; j++) {
        if (!rv[j]) continue;
        const double dx = wx[i] - rx[j], dy = wy[i] - ry[j], dd = dx * dx + dy * dy;
        if (dd > max_d2) continue;
        if (best == -1 || dd < bd) { best = j; bd = dd; }
      }
      if (best == -1 || best == 0 || best == n - 1) continue;
      const int up = next_valid_up(rv, n, best), dn = next_valid_down(rv, best);
      int other;
      if (up == -1 && dn == -1) continue;
      if (up == -1) other = dn;
      else if (dn == -1) other = up;
      else {
        const double du = (wx[i] - rx[up]) * (wx[i] - rx[up]) + (wy[i] - ry[up]) * (wy[i] - ry[up]);
        const double dd = (wx[i] - rx[dn]) * (wx[i] - rx[dn]) + (wy[i] - ry[dn]) * (wy[i] - ry[dn]);
        other = du < dd ? up : dn;
      }
      j1[i] = best; j2[i] = other; d2[i] = bd;
    }
    if (P->outliers_remove_doubles) {
      for (int j = 0; j < n; j++) dj[j] = 1e300;
      for (int i = 0; i < n; i++) if (j1[i] >= 0 && d2[i] < dj[j1[i]]) dj[j1[i]] = d2[i];
      for (int i = 0; i < n; i++) if (j1[i] >= 0 && d2[i] > 3.0 * dj[j1[i]]) j1[i] = -1;
    }
    int k = 0;
    for (int i = 0; i < n; i++) {
      if (j1[i] < 0) continue;
      const double a[2] = {rx[j1[i]], ry[j1[i]]}, b[2] = {rx[j2[i]], ry[j2[i]]}, x[2] = {wx[i], wy[i]};
      ds[i] = P->use_point_to_line_distance ? dist_to_segment(a, b, x) : sqrt(d2[i]);
      sorted[k++] = ds[i];
    }
    if (k > 0) {
      qsort(sorted, k, sizeof(double), cmp_double);
      int o1 = (int)floor(k * P->outliers_maxPerc), o2 = (int)floor(k * P->outliers_adaptive_order);
      if (o1 < 0) o1 = 0;
      if (o1 > k - 1) o1 = k - 1;
      if (o2 < 0) o2 = 0;
      if (o2 > k - 1) o2 = k - 1;
      const double lim = fmin(sorted[o1], P->outliers_adaptive_mult * sorted[o2]);
      error = 0; nvalid = 0;
      for (int i = 0; i < n; i++) {
        if (j1[i] < 0) continue;
        if (ds[i] > lim) j1[i] = -1;
        else { error += ds[i]; nvalid++; }
      }
    } else { nvalid = 0; error = 0; }
    if (nvalid < 5) { ok = 0; break; }
    double M[16] = {0}, g[4] = {0};
    for (int i = 0; i < n; i++) {
      if (j1[i] < 0) continue;
      double C[4] = {1, 0, 0, 1};
      if (P->use_point_to_line_distance) {
        const double ex = rx[j1[i]] - rx[j2[i]], ey = ry[j1[i]] - ry[j2[i]];
        const double inv = 1.0 / sqrt(ex * ex + ey * ey);
        const double ca = ey * inv, sa = -ex * inv; /* unit normal of the segment */
        C[0] = ca * ca; C[1] = ca * sa; C[2] = ca * sa; C[3] = sa * sa;
      }
      const double Mk[8] = {1, 0, sx[i], -sy[i], 0, 1, sy[i], sx[i]};
      const double qx = rx[j1[i]], qy = ry[j1[i]];
      double CM[8];
      for (int col = 0; col < 4; col++) { CM[col] = C[0] * Mk[col] + C[1] * Mk[4 + col]; CM[4 + col] = C[2] * Mk[col] + C[3] * Mk[4 + col]; }
      for (int r = 0; r < 4; r++)
        for (int col = 0; col < 4; col++) M[4 * r + col] += Mk[r] * CM[col] + Mk[4 + r] * CM[4 + col];
      for (int r = 0; r < 4; r++) g[r] += -2.0 * (qx * CM[r] + qy * CM[4 + r]);
    }
    /* a failed solve leaves x_new at the last accepted estimate (the first guess if there is none) */
    double x_gpc[3];
    if (!gpc_solve(M, g, x_gpc)) { ok = 0; break; }
    x_new[0] = x_gpc[0]; x_new[1] = x_gpc[1]; x_new[2] = x_gpc[2];
    /* pose_diff(x_new, x_old): x_new expressed relative to x_old */
    const double ddx = x_new[0] - x_old[0], ddy = x_new[1] - x_old[1];
    const double co = cos(x_old[2]), so = sin(x_old[2]);
    const double lx = co * ddx + so * ddy, ly = -so * ddx + co * ddy;
    double dth = x_new[2] - x_old[2];
    while (dth > M_PI) dth -= 2 * M_PI;
    while (dth < -M_PI) dth += 2 * M_PI;
    const int done = sqrt(lx * lx + ly * ly) < P->epsilon_xy && fabs(dth) < P->epsilon_theta;
    x_old[0] = x_new[0]; x_old[1] = x_new[1]; x_old[2] = x_new[2];
    if (done) { it++; break; }
  }
  out->x[0] = x_new[0]; out->x[1] = x_new[1]; out->x[2] = x_new[2];
  out->valid = ok; out->iterations = it < P->max_iterations ? it : P->max_iterations;
  out->nvalid = nvalid; out->error = error;
  free(rx); free(ry); free(sx); free(sy); free(wx); free(wy); free(rv); free(sv); free(j1); free(j2); free(d2); free(dj); free(ds); free(sorted);
  return ok;
}
