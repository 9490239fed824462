// K3 (lesson3) — the PL-ICP iteration loop of ONE scan pair, run by one CTA (sm_90a).  Shared by the pair kernel
// (plicp.cu: b2s_plicp_match) and the odometry node kernel (plicp_odometry.cu), so both run the same matcher.
//
// The algorithm (A. Censi, "An ICP variant using a point-to-line metric", ICRA 2008) with CSM's loop structure as
// selected by the parameters the reference sets: angular-window nearest-neighbour correspondences with the nearer
// index-neighbour as segment end, duplicate-correspondence pruning (3x rule), percentile / adaptive trimming on
// point-to-segment distances, closed-form point-to-line minimisation (GPC: Lagrange multiplier = largest real root of
// a quartic).  PARITY UNPINNED (DESIGN.md §7).
#pragma once

#include "common.cuh"

namespace b2s {

constexpr int ICP_THREADS = 256;

// shared memory per beam of one pair: rx ry sx sy wx wy d2 ds (double), dj (u64), j1 j2 (int), rv sv (u8)
constexpr size_t ICP_SMEM_PER_BEAM = 8 * 8 + 8 + 4 + 4 + 1 + 1;

__device__ inline double icp_quartic_largest_real_root(double c3, double c2, double c1, double c0) {
  // Durand-Kerner on the monic quartic, fixed 200 sweeps (deterministic), largest (numerically) real root
  double re[4] = {1.0, 0.4, -0.65, 0.0}, im[4] = {0.0, 0.9, 0.72, -0.85};
  const double scale = 1.0 + fmax(fmax(fabs(c3), fabs(c2)), fmax(fabs(c1), fabs(c0)));
  for (int k = 0; k < 4; k++) { re[k] *= scale; im[k] *= scale; }
  const double coef[4] = {c3, c2, c1, c0};
  for (int it = 0; it < 200; it++) {
    for (int k = 0; k < 4; k++) {
      double pr = 1.0, pi = 0.0;
      for (int q = 0; q < 4; q++) {
        const double nr = pr * re[k] - pi * im[k] + coef[q], ni = pr * im[k] + pi * re[k];
        pr = nr; pi = ni;
      }
      double dr = 1.0, di = 0.0;
      for (int j = 0; j < 4; j++) {
        if (j == k) continue;
        const double ar = re[k] - re[j], ai = im[k] - im[j];
        const double nr = dr * ar - di * ai, ni = dr * ai + di * ar;
        dr = nr; di = ni;
      }
      const double den = dr * dr + di * di;
      if (den == 0.0) continue;
      re[k] -= (pr * dr + pi * di) / den;
      im[k] -= (pi * dr - pr * di) / den;
    }
  }
  double best = -1e300;
  const double tol = 1e-7 * scale;
  bool found = false;
  for (int k = 0; k < 4; k++)
    if (fabs(im[k]) <= tol && (!found || re[k] > best)) { best = re[k]; found = true; }
  if (!found) {
    double bi = 1e300;
    for (int k = 0; k < 4; k++) if (fabs(im[k]) < bi) { bi = fabs(im[k]); best = re[k]; }
  }
  return best;
}

__device__ inline bool icp_gpc_solve(const double M[16], const double g[4], double x_out[3]) {
  const double A[4] = {M[0], M[1], M[4], M[5]}, B[4] = {M[2], M[3], M[6], M[7]}, Dm[4] = {M[10], M[11], M[14], M[15]};
  const double detA = A[0] * A[3] - A[1] * A[2];
  if (detA == 0.0) return false;
  const double Ai[4] = {A[3] / detA, -A[1] / detA, -A[2] / detA, A[0] / detA};
  const double AiB[4] = {Ai[0] * B[0] + Ai[1] * B[2], Ai[0] * B[1] + Ai[1] * B[3], Ai[2] * B[0] + Ai[3] * B[2], Ai[2] * B[1] + Ai[3] * B[3]};
  const double S[4] = {Dm[0] - (B[0] * AiB[0] + B[2] * AiB[2]), Dm[1] - (B[0] * AiB[1] + B[2] * AiB[3]),
                       Dm[2] - (B[1] * AiB[0] + B[3] * AiB[2]), Dm[3] - (B[1] * AiB[1] + B[3] * AiB[3])};
  const double Sa[4] = {S[3], -S[1], -S[2], S[0]};
  const double p = S[0] + S[3], q = S[0] * S[3] - S[1] * S[2];
  const double Aig1[2] = {Ai[0] * g[0] + Ai[1] * g[1], Ai[2] * g[0] + Ai[3] * g[1]};
  const double v[2] = {0.5 * ((B[0] * Aig1[0] + B[2] * Aig1[1]) - g[2]), 0.5 * ((B[1] * Aig1[0] + B[3] * Aig1[1]) - g[3])};
  const double Sav[2] = {Sa[0] * v[0] + Sa[1] * v[1], Sa[2] * v[0] + Sa[3] * v[1]};
  const double vv = v[0] * v[0] + v[1] * v[1], vSav = v[0] * Sav[0] + v[1] * Sav[1], vSa2v = Sav[0] * Sav[0] + Sav[1] * Sav[1];
  const double lam = icp_quartic_largest_real_root(2 * p, p * p + 2 * q - vv, 2 * p * q - 2 * vSav, q * q - vSa2v);
  const double den = lam * lam + p * lam + q;
  if (den == 0.0) return false;
  const double r[2] = {(Sav[0] + lam * v[0]) / den, (Sav[1] + lam * v[1]) / den};
  const double Br[2] = {B[0] * r[0] + B[1] * r[1] + 0.5 * g[0], B[2] * r[0] + B[3] * r[1] + 0.5 * g[1]};
  x_out[0] = -(Ai[0] * Br[0] + Ai[1] * Br[1]);
  x_out[1] = -(Ai[2] * Br[0] + Ai[3] * Br[1]);
  x_out[2] = atan2(r[1], r[0]);
  return isfinite(x_out[0]) && isfinite(x_out[1]) && isfinite(x_out[2]);
}

// One scan's LaserScanToLDP (plicp_odometry.cc:285-322) into a pair slot: beam i valid iff range_min < r < range_max,
// its point r (cos, sin)(theta_i) in the laser frame, (0, 0) when invalid.
__device__ __forceinline__ void icp_load_point(double r, double th, double range_min, double range_max, double *x,
                                               double *y, uint8_t *v, int i) {
  v[i] = r > range_min && r < range_max;
  x[i] = v[i] ? r * cos(th) : 0.0;
  y[i] = v[i] ? r * sin(th) : 0.0;
}

// The pair's working memory in shared memory (n beams each); `red`, `xs` and `s_cnt` are the reduction rows and the
// running estimate / counters every thread reads.
struct IcpPairSmem {
  const double *rx, *ry, *sx, *sy;  // reference and current scan points
  const uint8_t *rv, *sv;
  double *wx, *wy, *d2, *ds;
  unsigned long long *dj;  // min squared distance per reference beam
  int *j1, *j2;
  double (*red)[17];  // [ICP_THREADS][17]: 16 used; the odd pitch keeps the tree reduction off one bank group
  double *xs;         // [8]: x_old[3], x_new[3], lim, error
  int *s_cnt;         // [4]: k (valid before trim), nvalid, ok, done
};

// Carves the per-beam arrays (everything but the two scans' points) out of `dyn`, after the 2 * 2 * n doubles of the
// points: the layout of the pair kernel.
__device__ __forceinline__ void icp_carve(unsigned char *dyn, int n, double *&rx, double *&ry, double *&sx, double *&sy,
                                          uint8_t *&rv, uint8_t *&sv, IcpPairSmem &S) {
  rx = reinterpret_cast<double *>(dyn); ry = rx + n; sx = ry + n; sy = sx + n;
  S.wx = sy + n; S.wy = S.wx + n;
  S.d2 = S.wy + n; S.ds = S.d2 + n;
  S.dj = reinterpret_cast<unsigned long long *>(S.ds + n);
  S.j1 = reinterpret_cast<int *>(S.dj + n); S.j2 = S.j1 + n;
  rv = reinterpret_cast<uint8_t *>(S.j2 + n); sv = rv + n;
}

// sm_icp on the pair held in S, from `guess` (read by thread 0).  Every thread of the CTA calls it once the points are
// loaded (the first __syncthreads inside orders the loads); thread 0 writes `out`.  The caller synchronises before it
// reloads a slot or reads `out` from another thread.
__device__ inline void icp_pair(const b2s_icp_params &P, int n, double min_theta, double max_theta, const IcpPairSmem &S,
                                const double guess[3], b2s_icp_result *out) {
  const double *rx = S.rx, *ry = S.ry, *sx = S.sx, *sy = S.sy;
  const uint8_t *rv = S.rv, *sv = S.sv;
  double *wx = S.wx, *wy = S.wy, *d2 = S.d2, *ds = S.ds, *xs = S.xs;
  unsigned long long *dj = S.dj;
  int *j1 = S.j1, *j2 = S.j2, *s_cnt = S.s_cnt;
  double(*red)[17] = S.red;
  const int tid = threadIdx.x;
  const double PI = 3.14159265358979323846;
  if (tid == 0) {
    for (int q = 0; q < 3; q++) { xs[q] = guess[q]; xs[3 + q] = xs[q]; }
    s_cnt[2] = 1; s_cnt[3] = 0;
  }
  __syncthreads();
  const double ang_res = (max_theta - min_theta) / n;
  const double max_d2 = P.max_correspondence_dist * P.max_correspondence_dist;
  int it = 0;
  for (it = 0; it < P.max_iterations; it++) {
    const double x0 = xs[0], x1 = xs[1], x2 = xs[2];
    const double c = cos(x2), s = sin(x2);
    // ---- 1+2: transform, correspondences ----
    for (int i = tid; i < n; i += ICP_THREADS) {
      const double px = c * sx[i] - s * sy[i] + x0, py = s * sx[i] + c * sy[i] + x1;
      wx[i] = px; wy[i] = py;
      int best = -1, other = -1;
      double bd = 0.0;
      if (sv[i]) {
        const double nrm = sqrt(px * px + py * py);
        const double delta = fabs(P.max_angular_correction_deg * PI / 180.0) + fabs(atan(P.max_linear_correction / nrm));
        const int range = (int)ceil(delta / ang_res);
        double st = atan2(py, px);
        if (st < min_theta) st += 2 * PI;
        if (st > max_theta) st -= 2 * PI;
        const double start_cell = (st - min_theta) / (max_theta - min_theta) * n;
        int from = (int)floor(start_cell - range), to = (int)ceil(start_cell + range);
        from = min(max(from, 0), n - 1);
        to = min(max(to, 0), n - 1);
        for (int j = from; j <= to; j++) {
          if (!rv[j]) continue;
          const double dx = px - rx[j], dy = py - ry[j], dd = dx * dx + dy * dy;
          if (dd > max_d2) continue;
          if (best == -1 || dd < bd) { best = j; bd = dd; }
        }
        if (best == 0 || best == n - 1) best = -1;
        if (best != -1) {
          int up = -1, dn = -1;
          for (int k = best + 1; k < n; k++) if (rv[k]) { up = k; break; }
          for (int k = best - 1; k >= 0; k--) if (rv[k]) { dn = k; break; }
          if (up == -1 && dn == -1) best = -1;
          else if (up == -1) other = dn;
          else if (dn == -1) other = up;
          else {
            const double du = (px - rx[up]) * (px - rx[up]) + (py - ry[up]) * (py - ry[up]);
            const double dd = (px - rx[dn]) * (px - rx[dn]) + (py - ry[dn]) * (py - ry[dn]);
            other = du < dd ? up : dn;
          }
        }
      }
      j1[i] = best; j2[i] = other; d2[i] = bd;
      dj[i] = 0x7ff0000000000000ull;  // +inf
    }
    __syncthreads();
    // ---- 3: duplicates ----
    if (P.outliers_remove_doubles) {
      for (int i = tid; i < n; i += ICP_THREADS)
        if (j1[i] >= 0) atomicMin(&dj[j1[i]], (unsigned long long)__double_as_longlong(d2[i]));
      __syncthreads();
      for (int i = tid; i < n; i += ICP_THREADS)
        if (j1[i] >= 0 && d2[i] > 3.0 * __longlong_as_double((long long)dj[j1[i]])) j1[i] = -1;
      __syncthreads();
    }
    // ---- 4: trimming ----
    if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; xs[6] = 0.0; xs[7] = 0.0; }
    for (int i = tid; i < n; i += ICP_THREADS) {
      if (j1[i] < 0) continue;
      double dist;
      if (P.use_point_to_line_distance) {
        const double ax = rx[j1[i]], ay = ry[j1[i]], ex = rx[j2[i]] - ax, ey = ry[j2[i]] - ay;
        const double len2 = ex * ex + ey * ey;
        double t = len2 > 0 ? ((wx[i] - ax) * ex + (wy[i] - ay) * ey) / len2 : 0.0;
        t = fmin(fmax(t, 0.0), 1.0);
        const double qx = ax + t * ex - wx[i], qy = ay + t * ey - wy[i];
        dist = sqrt(qx * qx + qy * qy);
      } else {
        dist = sqrt(d2[i]);
      }
      ds[i] = dist;
    }
    __syncthreads();
    int my_valid = 0;
    for (int i = tid; i < n; i += ICP_THREADS) my_valid += j1[i] >= 0;
    if (my_valid) atomicAdd(&s_cnt[0], my_valid);
    __syncthreads();
    const int k = s_cnt[0];
    if (k > 0) {
      int o1 = (int)floor(k * P.outliers_maxPerc), o2 = (int)floor(k * P.outliers_adaptive_order);
      o1 = min(max(o1, 0), k - 1);
      o2 = min(max(o2, 0), k - 1);
      // rank of each valid distance among the valid ones (ties broken by index) = its position after sorting
      for (int i = tid; i < n; i += ICP_THREADS) {
        if (j1[i] < 0) continue;
        const double v = ds[i];
        int rank = 0;
        for (int j = 0; j < n; j++) rank += (j1[j] >= 0) && (ds[j] < v || (ds[j] == v && j < i));
        if (rank == o1) xs[6] = v;
        if (rank == o2) xs[7] = v;
      }
      __syncthreads();
      const double lim = fmin(xs[6], P.outliers_adaptive_mult * xs[7]);
      __syncthreads();
      for (int i = tid; i < n; i += ICP_THREADS)
        if (j1[i] >= 0 && ds[i] > lim) j1[i] = -1;
    }
    __syncthreads();
    // ---- 5: accumulate the 4x4 system (per-thread partials in beam order, then a fixed-order tree) ----
    double acc[20];
#pragma unroll
    for (int q = 0; q < 20; q++) acc[q] = 0.0;  // 10 upper-triangular M entries, 4 g entries, error, count
    for (int i = tid; i < n; i += ICP_THREADS) {
      if (j1[i] < 0) continue;
      double C0 = 1, C1 = 0, C3 = 1;
      if (P.use_point_to_line_distance) {
        const double ex = rx[j1[i]] - rx[j2[i]], ey = ry[j1[i]] - ry[j2[i]];
        const double inv = 1.0 / sqrt(ex * ex + ey * ey);
        const double ca = ey * inv, sa = -ex * inv;
        C0 = ca * ca; C1 = ca * sa; C3 = sa * sa;
      }
      const double Mk[8] = {1, 0, sx[i], -sy[i], 0, 1, sy[i], sx[i]};
      double CM[8];
      for (int col = 0; col < 4; col++) { CM[col] = C0 * Mk[col] + C1 * Mk[4 + col]; CM[4 + col] = C1 * Mk[col] + C3 * Mk[4 + col]; }
      int w = 0;
      for (int r = 0; r < 4; r++)
        for (int col = r; col < 4; col++) acc[w++] += Mk[r] * CM[col] + Mk[4 + r] * CM[4 + col];
      const double qx = rx[j1[i]], qy = ry[j1[i]];
      for (int r = 0; r < 4; r++) acc[10 + r] += -2.0 * (qx * CM[r] + qy * CM[4 + r]);
      acc[14] += ds[i];
      acc[15] += 1.0;
    }
#pragma unroll
    for (int q = 0; q < 16; q++) red[tid][q] = acc[q];
    __syncthreads();
    for (int d = ICP_THREADS / 2; d > 0; d >>= 1) {
      if (tid < d)
        for (int q = 0; q < 16; q++) red[tid][q] += red[tid + d][q];
      __syncthreads();
    }
    if (tid == 0) {
      const int nvalid = (int)red[0][15];
      s_cnt[1] = nvalid;
      xs[7] = red[0][14];
      bool ok = nvalid >= 5;
      double xn[3] = {xs[3], xs[4], xs[5]};
      if (ok) {
        double M[16], g[4];
        int w = 0;
        for (int r = 0; r < 4; r++)
          for (int col = r; col < 4; col++) { M[4 * r + col] = red[0][w]; M[4 * col + r] = red[0][w]; w++; }
        for (int r = 0; r < 4; r++) g[r] = red[0][10 + r];
        ok = icp_gpc_solve(M, g, xn);
      }
      if (!ok) {
        s_cnt[2] = 0;
        s_cnt[3] = 1;
      } else {
        const double ddx = xn[0] - xs[0], ddy = xn[1] - xs[1];
        const double co = cos(xs[2]), so = sin(xs[2]);
        const double lx = co * ddx + so * ddy, ly = -so * ddx + co * ddy;
        double dth = xn[2] - xs[2];
        while (dth > PI) dth -= 2 * PI;
        while (dth < -PI) dth += 2 * PI;
        s_cnt[3] = (sqrt(lx * lx + ly * ly) < P.epsilon_xy && fabs(dth) < P.epsilon_theta) ? 2 : 0;
        for (int q = 0; q < 3; q++) { xs[3 + q] = xn[q]; xs[q] = xn[q]; }
      }
    }
    __syncthreads();
    if (s_cnt[3] == 1) break;              // failed: iterations = it
    if (s_cnt[3] == 2) { it++; break; }    // converged
  }
  if (tid == 0) {
    b2s_icp_result &r = *out;
    r.x[0] = xs[3]; r.x[1] = xs[4]; r.x[2] = xs[5];
    r.error = xs[7];
    r.valid = s_cnt[2];
    r.iterations = min(it, P.max_iterations);
    r.nvalid = s_cnt[1];
    r.reserved = 0;
  }
}

}  // namespace b2s
