/* TEST INFRASTRUCTURE — CPU restatement of lesson5's whole de-skew node over one recording (LidarUndistortion,
 * lesson5/src/lidar_undistortion.cc): the callbacks (:82-159), PruneImuDeque (:177-249), PruneOdomDeque (:252-336),
 * CorrectLaserScan (:339-393) and ResetParameters (:60-79), with the node's members as state.  Built on the per-scan
 * restatements of deskew_oracle.c (orc_deskew_integrate_imu, orc_deskew_odom_increment, orc_deskew_scan), linked into a
 * library of its own (oracle/deskew_node_port.py).  Pinned to the unmodified node by tests/test_deskew_node_reference.py
 * except tf's quaternionMsgToTF and Matrix3x3::getRPY, which are linear_math.h's, as the node's stand-in
 * (oracle/shim/tf2/LinearMath/Transform.h) restates them: tf is not in the reference tree.
 *
 * The node's AsyncSpinner runs the IMU, odometry and scan callbacks under separate locks, so what a scan callback sees
 * is the number of messages of each log delivered before it (imu_arrived / odom_arrived). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "linear_math.h"

typedef struct {
  double time_start, time_increment;
  float range_min, range_max;
  int32_t use_imu, use_odom;
  int32_t imu_last, pad_;
  double odom_start_time, odom_end_time;
  float odom_incre[3];
  float pad2_;
} orc_deskew_scan_info; /* as in deskew_oracle.c: the layout of b2s_deskew_scan */

typedef struct { uint32_t sec, nsec; double angular_velocity[3]; } orc_imu_msg;
typedef struct { uint32_t sec, nsec; double position[3], orientation[4]; } orc_odom_msg;
typedef struct {
  uint32_t sec, nsec;
  float time_increment, range_min, range_max;
  int32_t imu_arrived, odom_arrived, reserved;
} orc_node_scan;

int32_t orc_deskew_integrate_imu(int n_imu, const double *stamp, const double *ang_vel, double scan_start, double scan_end,
                                 int cap, double *imu_time, double *rx, double *ry, double *rz);
void orc_deskew_odom_increment(const double start[6], const double end[6], float out[3]);
void orc_deskew_scan(int n_beams, const float *ranges, double angle_min, double angle_increment, const orc_deskew_scan_info *s,
                     const double *imu_time, const double *rx, const double *ry, const double *rz, float *out_xyz);

enum { PUBLISHED = 0, HELD = 1, WAIT_IMU = 2, IMU_EMPTY = 3, WAIT_ODOM = 4, ODOM_EMPTY = 5, UNDEFINED = 6 };
#define QUEUE_LENGTH 2000 /* queueLength (:20) */

static void pose_of(const orc_odom_msg *m, double out[6]) {
  static const orc_odom_msg none; /* nav_msgs::Odometry(): stamp 0, position 0, quaternion (0, 0, 0, 0) */
  if (!m) m = &none;
  out[0] = m->position[0];
  out[1] = m->position[1];
  out[2] = m->position[2];
  orc_tf t; /* tf::quaternionMsgToTF, then tf::Matrix3x3(q).getRPY */
  tf_set_rotation(&t, m->orientation);
  tf_get_rpy(&t, &out[3], &out[4], &out[5]);
}

/* One recording through the node.  Per scan j: out_status[j]; out_state[j] (zero unless published or undefined);
 * out_xyz[j] (the published cloud, else zero); out_poses[j][12] (may be NULL): the start and end odometry pose the
 * node's getRPY gives; out_imu[j][4][2000] (may be NULL): the node's IMU table (time, rot x, y, z) when it corrected
 * scan j.  Returns 0, or -1 when out of memory. */
int orc_deskew_node(int use_imu, int use_odom, float angle_min, float angle_increment, int n_beams, int n_scans,
                    const orc_node_scan *scans, const float *ranges, int n_imu, const orc_imu_msg *imu, int n_odom,
                    const orc_odom_msg *odom, int32_t *out_status, orc_deskew_scan_info *out_state, float *out_xyz,
                    double *out_poses, double *out_imu) {
  double *imu_t = malloc(sizeof(double) * (size_t)(n_imu > 0 ? n_imu : 1));
  double *imu_w = malloc(sizeof(double) * 3 * (size_t)(n_imu > 0 ? n_imu : 1));
  double *odom_t = malloc(sizeof(double) * (size_t)(n_odom > 0 ? n_odom : 1));
  double *tab = calloc(8 * QUEUE_LENGTH, sizeof(double)); /* the node's imu_time_ / imu_rot_*_ members, then scratch */
  if (!imu_t || !imu_w || !odom_t || !tab) {
    free(imu_t); free(imu_w); free(odom_t); free(tab);
    return -1;
  }
  double *mt = tab, *mx = tab + QUEUE_LENGTH, *my = tab + 2 * QUEUE_LENGTH, *mz = tab + 3 * QUEUE_LENGTH;
  double *st = tab + 4 * QUEUE_LENGTH, *sx = st + QUEUE_LENGTH, *sy = st + 2 * QUEUE_LENGTH, *sz = st + 3 * QUEUE_LENGTH;
  for (int i = 0; i < n_imu; i++) {
    imu_t[i] = ros_time_to_sec(imu[i].sec, imu[i].nsec);
    memcpy(imu_w + 3 * i, imu[i].angular_velocity, sizeof(double) * 3);
  }
  for (int i = 0; i < n_odom; i++) odom_t[i] = ros_time_to_sec(odom[i].sec, odom[i].nsec);
  const double scan_count = (double)n_beams;
  int ilo = 0, olo = 0, start_msg = -1, end_msg = -1;
  memset(out_xyz, 0, sizeof(float) * 3 * (size_t)n_beams * (size_t)n_scans);
  for (int j = 0; j < n_scans; j++) {
    orc_deskew_scan_info s;
    memset(&s, 0, sizeof s);
    double poses[12] = {0};
    int status = PUBLISHED;
    if (out_imu) memset(out_imu + (size_t)j * 4 * QUEUE_LENGTH, 0, sizeof(double) * 4 * QUEUE_LENGTH);
    if (j == n_scans - 1) {
      status = HELD; /* CacheLaserScan (:145-150): scan j is popped at the callback of scan j + 1 */
      goto done;
    }
    const orc_node_scan *sc = &scans[j], *next = &scans[j + 1];
    const double start = ros_time_to_sec(sc->sec, sc->nsec), inc = sc->time_increment, end = start + inc * (scan_count - 1);
    s.time_start = start;
    s.time_increment = inc;
    s.range_min = sc->range_min;
    s.range_max = sc->range_max;
    s.use_imu = use_imu != 0;
    s.use_odom = use_odom != 0;
    if (use_imu) {
      const int hi = next->imu_arrived;
      if (ilo == hi || imu_t[ilo] > start || imu_t[hi - 1] < end) { status = WAIT_IMU; goto done; }
      while (ilo < hi && imu_t[ilo] < start - 0.1) ++ilo;
      if (ilo == hi) { status = IMU_EMPTY; goto done; }
      s.imu_last = orc_deskew_integrate_imu(hi - ilo, imu_t + ilo, imu_w + 3 * (size_t)ilo, start, end, QUEUE_LENGTH, st, sx, sy, sz);
      if (s.imu_last == -2) {
        status = UNDEFINED; /* the node's table after this is not modelled */
      } else {
        for (int i = 0; i <= s.imu_last; i++) { mt[i] = st[i]; mx[i] = sx[i]; my[i] = sy[i]; mz[i] = sz[i]; }
      }
    }
    if (use_odom) {
      const int hi = next->odom_arrived;
      if (olo == hi || odom_t[olo] > start || odom_t[hi - 1] < end) { if (status == PUBLISHED) status = WAIT_ODOM; goto done; }
      while (olo < hi && odom_t[olo] < start - 0.1) ++olo;
      if (olo == hi) { if (status == PUBLISHED) status = ODOM_EMPTY; goto done; }
      for (int i = olo; i < hi; i++) {
        if (odom_t[i] < start) { start_msg = i; continue; }
        if (odom_t[i] <= end) end_msg = i;
        else break;
      }
      pose_of(start_msg < 0 ? NULL : &odom[start_msg], poses);
      pose_of(end_msg < 0 ? NULL : &odom[end_msg], poses + 6);
      s.odom_start_time = start_msg < 0 ? 0.0 : odom_t[start_msg];
      s.odom_end_time = end_msg < 0 ? 0.0 : odom_t[end_msg];
      orc_deskew_odom_increment(poses, poses + 6, s.odom_incre);
    }
    if (status == PUBLISHED) {
      orc_deskew_scan(n_beams, ranges + (size_t)j * n_beams, angle_min, angle_increment, &s, mt, mx, my, mz,
                      out_xyz + (size_t)j * n_beams * 3);
      if (out_imu) {
        double *o = out_imu + (size_t)j * 4 * QUEUE_LENGTH;
        memcpy(o, mt, sizeof(double) * QUEUE_LENGTH);
        memcpy(o + QUEUE_LENGTH, mx, sizeof(double) * QUEUE_LENGTH);
        memcpy(o + 2 * QUEUE_LENGTH, my, sizeof(double) * QUEUE_LENGTH);
        memcpy(o + 3 * QUEUE_LENGTH, mz, sizeof(double) * QUEUE_LENGTH);
      }
    }
    if (status == PUBLISHED || status == UNDEFINED) memset(tab, 0, sizeof(double) * 4 * QUEUE_LENGTH); /* ResetParameters */
  done:
    out_status[j] = status;
    if (status != PUBLISHED && status != UNDEFINED) memset(&s, 0, sizeof s);
    if (out_state) out_state[j] = s;
    if (out_poses) memcpy(out_poses + 12 * (size_t)j, poses, sizeof poses);
  }
  free(imu_t); free(imu_w); free(odom_t); free(tab);
  return 0;
}
