/*
 * plicp_odometry_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of lesson3's odometry node, ScanMatchPLICP (reference/lesson3/src/plicp_odometry.cc:191-517): the
 * node's loop in C around the PL-ICP restatement orc_plicp_match (oracle/plicp_oracle.c).  Built with it into a library
 * of its own (oracle/plicp_odometry_port.py), built by oracle/recipes.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200slam.h"
#include "linear_math.h"

int orc_plicp_match(const b2s_icp_params *P, int n, const double *ref_r, const double *sens_r, const double *theta,
                    double range_min, double range_max, const double first_guess[3], b2s_icp_result *out);

/* The node's loop for ONE recording from a fresh node, in C around orc_plicp_match.  tf2's LinearMath and ros::Duration
 * are linear_math.h's, in double without FMA contraction.  After a failed match the node tests NewKeyframeNeeded on a
 * default-constructed (uninitialised) tf2::Transform; here it is the identity (DESIGN.md §7).  The unmodified node,
 * compiled against the stand-ins under oracle/shim/ (oracle/ref_lesson3.cpp), pins this restatement bit for bit. */
static double tf_yaw_of(const orc_tf *t) {
  double q[4];
  tf_get_rotation(t, q);
  return tf2_get_yaw(q);
}
/* ScanMatchPLICP::CreateTfFromXYTheta: origin (x, y, 0), rotation Quaternion::setRPY(0, 0, theta) */
static orc_tf tf_from_xyt(double x, double y, double theta) {
  double q[4];
  quat_set_rpy(0.0, 0.0, theta, q);
  orc_tf t;
  t.o[0] = x; t.o[1] = y; t.o[2] = 0.0;
  tf_set_rotation(&t, q);
  return t;
}

/* ranges [n_scans][n] float32, stamps [n_scans][2] (sec, nsec) -> out [n_scans] as b2s_plicp_odom_process fills it */
void orc_plicp_odometry(const b2s_plicp_odom_params *P, int n, float angle_min, float angle_increment, float range_min,
                        float range_max, int n_scans, const float *ranges, const uint32_t *stamps,
                        b2s_plicp_odom_step *out) {
  double *theta = malloc(sizeof(double) * n), *kf = malloc(sizeof(double) * n), *cur = malloc(sizeof(double) * n);
  for (int i = 0; i < n; i++) theta[i] = (double)(angle_min + (float)i * angle_increment); /* :308 */
  orc_tf b2l, l2b, bio, bio_kf;
  b2l.o[0] = P->base_to_laser[0]; b2l.o[1] = P->base_to_laser[1]; b2l.o[2] = P->base_to_laser[2];
  tf_set_rotation(&b2l, P->base_to_laser + 3);
  l2b = tf_inverse(&b2l);
  tf_identity(&bio);
  tf_identity(&bio_kf);
  double vx = 0.0, vaz = 0.0;
  uint32_t last_sec = 0, last_nsec = 0;
  int scan_count = 0, kf_scan = 0;
  for (int s = 0; s < n_scans; s++) {
    const float *r = ranges + (size_t)s * n;
    b2s_plicp_odom_step *o = out + s;
    memset(o, 0, sizeof *o);
    if (s == 0) {
      for (int i = 0; i < n; i++) kf[i] = r[i];
      last_sec = stamps[0]; last_nsec = stamps[1];
      o->orientation[3] = 1.0; o->keyframe = 1; o->reference_scan = -1;
      continue;
    }
    for (int i = 0; i < n; i++) cur[i] = r[i];
    const double dt = ros_duration_to_sec(ros_time_diff(stamps[2 * s], stamps[2 * s + 1], last_sec, last_nsec));
    const double pr_x = vx < 1e-6 ? 0.0 : dt * vx;
    orc_tf pc = tf_from_xyt(pr_x, 0.0, 0.0);
    orc_tf kfi = tf_inverse(&bio_kf), rel = tf_mul(&bio, &kfi);
    pc = tf_mul(&pc, &rel);
    orc_tf bioi = tf_inverse(&bio), t1 = tf_mul(&l2b, &bioi), t2 = tf_mul(&t1, &pc), t3 = tf_mul(&t2, &bio);
    orc_tf pcl = tf_mul(&t3, &b2l);
    const double guess[3] = {pcl.o[0], pcl.o[1], tf_yaw_of(&pcl)};
    b2s_icp_result res;
    orc_plicp_match(&P->icp, n, kf, cur, theta, (double)range_min, (double)range_max, guess, &res);
    orc_tf corr;
    tf_identity(&corr);
    if (res.valid) {
      orc_tf cl = tf_from_xyt(res.x[0], res.x[1], res.x[2]), u = tf_mul(&b2l, &cl);
      corr = tf_mul(&u, &l2b);
      bio = tf_mul(&bio_kf, &corr);
      vx = corr.o[0] / dt;
      vaz = tf_yaw_of(&corr) / dt;
    }
    for (int q = 0; q < 3; q++) { o->position[q] = bio.o[q]; o->first_guess[q] = guess[q]; }
    tf_get_rotation(&bio, o->orientation);
    o->linear[0] = vx;
    o->angular[2] = vaz;
    o->icp = res;
    o->published = 1;
    o->reference_scan = kf_scan;
    int promote;
    scan_count++;
    if (fabs(tf_yaw_of(&corr)) > P->kf_dist_angular) promote = 1;
    else if (scan_count == P->kf_scan_count) { scan_count = 0; promote = 1; }
    else promote = corr.o[0] * corr.o[0] + corr.o[1] * corr.o[1] > P->kf_dist_linear * P->kf_dist_linear;
    if (promote) {
      memcpy(kf, cur, sizeof(double) * n);
      bio_kf = bio;
      kf_scan = s;
    }
    o->keyframe = promote;
    last_sec = stamps[2 * s]; last_nsec = stamps[2 * s + 1];
  }
  free(theta); free(kf); free(cur);
}
