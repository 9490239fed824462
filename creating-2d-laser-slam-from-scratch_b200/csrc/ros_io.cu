// ROS-shaped input adapters (host C++, no device work): the conversions the lesson nodes apply to sensor_msgs/LaserScan
// fields before the hot path sees them (SURVEY.md §8(f).4).  ROS itself is out of scope.
//   SlamKarto::getLaser / addScan                       lesson6/src/karto_slam.cc:323-395, 407-434
//   LaserRangeFinder::SetRangeThreshold / Update        lesson6/lib/open_karto/include/open_karto/Karto.h:3778-3787, 4152-4161
//   HectorMappingRos::rosPointCloudToDataContainer      lesson4/src/hector_mapping/hector_slam.cc:320-362
//   HectorMappingRos::scanCallback (projectLaser + the above, per-beam arithmetic in hector_scan.cuh)   :186-205
#include <cmath>
#include <vector>

#include "common.cuh"
#include "hector_scan.cuh"
#include "karto_internal.cuh"

using namespace b2s;

namespace b2s {

// getLaser's setters without any reading-count check (b2s_karto_node_create uses it too)
b2s_status karto_laser_from_msg(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                                b2s_laser *out) {
  if (!scan || !laser_pose_in_base || !out) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  // the setters take kt_double: the float32 message fields widen exactly
  const double min_angle = scan->angle_min, max_angle = scan->angle_max, res = scan->angle_increment;
  const double min_range = scan->range_min, max_range = scan->range_max;
  if (!(res != 0.0)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "angle_increment is zero");
  out->min_angle = min_angle;
  out->angular_resolution = res;
  out->min_range = min_range;
  out->max_range = max_range;
  // math::Clip(rangeThreshold, min, max) (Karto.h:3781)
  out->range_threshold = use_scan_range < min_range ? min_range : (use_scan_range > max_range ? max_range : use_scan_range);
  out->offset_pose[0] = laser_pose_in_base[0];
  out->offset_pose[1] = laser_pose_in_base[1];
  out->offset_pose[2] = laser_pose_in_base[2];
  out->n_readings = (int32_t)cast_u32(kround((max_angle - min_angle) / res));  // Update(): no + 1
  out->reserved = 0;
  return B2S_OK;
}

}  // namespace b2s

extern "C" {

b2s_status b2s_ros_karto_laser(const b2s_laser_scan_msg *scan, const double laser_pose_in_base[3], double use_scan_range,
                               b2s_laser *out) {
  if (b2s_status st = karto_laser_from_msg(scan, laser_pose_in_base, use_scan_range, out)) return st;
  if (out->n_readings != scan->n_ranges)
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "LaserScan carries a different number of ranges than Round((angle_max - angle_min) / angle_increment): "
                                 "this function requires the two to be equal");
  return B2S_OK;
}

b2s_status b2s_ros_karto_readings(const b2s_laser_scan_msg *scan, int inverted, double *out) {
  if (!scan || !out || (scan->n_ranges > 0 && !scan->ranges)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  const int n = scan->n_ranges;
  for (int i = 0; i < n; i++) out[i] = (double)scan->ranges[inverted ? n - 1 - i : i];
  return B2S_OK;
}

b2s_status b2s_ros_hector_points(const float *pts, int n, const float laser_in_base[4], float scale_to_map, float min_dist,
                                 float max_dist, double use_max_scan_range, float z_min, float z_max, float *out_points,
                                 float out_origo[2], int32_t *out_n) {
  if (!laser_in_base || !out_origo || !out_n || n < 0 || (n > 0 && (!pts || !out_points))) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  const HectorBeamFilter f = hector_scan_filter(laser_in_base, scale_to_map, min_dist, max_dist, use_max_scan_range, z_min, z_max);
  out_origo[0] = (float)f.mount.o[0] * scale_to_map;  // Eigen::Vector2f(laserPos.x(), laserPos.y()) * scaleToMap
  out_origo[1] = (float)f.mount.o[1] * scale_to_map;
  int k = 0;
  for (int i = 0; i < n; i++) {
    float x, y;
    if (!hector_node_filter_point(f, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], x, y)) continue;
    out_points[2 * k] = x;
    out_points[2 * k + 1] = y;
    k++;
  }
  *out_n = k;
  return B2S_OK;
}

b2s_status b2s_ros_hector_scans(const b2s_laser_scan_msg *geometry, const b2s_hector_scan_filter *filter, float scale_to_map,
                                int n_scans, const float *ranges, float *out_points, int32_t *out_n_points,
                                float out_origo[2]) {
  if (!geometry || !filter || !out_origo || n_scans < 0 || geometry->n_ranges < 0 || (n_scans > 0 && !out_n_points))
    B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument or negative count");
  const int n = geometry->n_ranges;
  if (n_scans > 0 && n > 0 && (!ranges || !out_points)) B2S_FAIL(B2S_ERR_BAD_PARAMS, "null argument");
  const b2s_hector_scan_filter &q = *filter;
  const HectorBeamFilter f = hector_scan_filter(q.laser_in_base, scale_to_map, q.min_dist, q.max_dist, q.use_max_scan_range,
                                                q.z_min, q.z_max);
  const double cutoff = hector_range_cutoff(q.range_cutoff, geometry->range_max);
  std::vector<double> unit(2 * (size_t)n);
  hector_unit_vectors(geometry->angle_min, geometry->angle_increment, n, unit.data());
  out_origo[0] = (float)f.mount.o[0] * scale_to_map;
  out_origo[1] = (float)f.mount.o[1] * scale_to_map;
  size_t k = 0;
  for (int s = 0; s < n_scans; s++) {
    const float *r = ranges + (size_t)s * n;
    const size_t k0 = k;
    for (int i = 0; i < n; i++) {
      float x, y;
      if (!hector_node_beam(f, r[i], unit[2 * i], unit[2 * i + 1], cutoff, geometry->range_min, x, y)) continue;
      out_points[2 * k] = x;
      out_points[2 * k + 1] = y;
      k++;
    }
    out_n_points[s] = (int32_t)(k - k0);
  }
  return B2S_OK;
}

}  // extern "C"
