// lesson4's LaserScan -> DataContainer conversion, per beam, in one definition: the host adapters (ros_io.cu:
// b2s_ros_hector_points, b2s_ros_hector_scans) and the ingest stage of the batched stream kernel (hector_slam.cu:
// k_hs_stream_batch<_, true>, behind b2s_hector_slam_process_scans_batch and the node handle, hector_node.cu) all apply
// it with a HectorBeamFilter, whose mount is a full tf::Transform.
// HectorMappingRos::scanCallback (lesson4/src/hector_mapping/hector_slam.cc:186-205) does two things to a scan:
//   projector_.projectLaser(scan, cloud, 30.0)     laser_geometry's LaserProjection (not in the reference tree, see
//                                                  DESIGN §7: restated from the package's published behaviour)
//   rosPointCloudToDataContainer                    hector_slam.cc:320-362 (pinned by tests/test_ros_io.py)
// Only IEEE multiply / add / compare / convert here: the transcendental values (the beams' unit vectors, the mount's
// basis) are the host C library's, computed by the caller and passed in, so the device and the host adapter
// produce the same points bit for bit under the library's -fmad=false.
#pragma once
#include <cmath>

#include "common.cuh"
#include "ros_math.cuh"

namespace b2s {

// LaserProjection::projectLaser (sensor_msgs::PointCloud form) on beam i: kept iff range < cutoff (double) and
// range >= range_min (float); NaN and +-inf drop out.  Point32 x / y = (float)(range * unit vector), z = 0.
__host__ __device__ __forceinline__ bool hector_project_beam(float range, double ux, double uy, double cutoff, float range_min,
                                                             float &x, float &y) {
  if (!(((double)range < cutoff) && (range >= range_min))) return false;
  x = (float)((double)range * ux);
  y = (float)((double)range * uy);
  return true;
}

// The settings of rosPointCloudToDataContainer: the tf::StampedTransform of the laser mount (base_link <- laser,
// tfScalar = double) and the squared distance window.  The node handle (hector_node.cu) builds one per node from its
// parameters; hector_scan_filter builds one from b2s_hector_scan_filter's.
struct HectorBeamFilter {
  float sqr_min, sqr_max;
  double use_max_scan_range;
  TfTransform mount;
  float z_min, z_max;
  float scale_to_map;
};

// b2s_hector_scan_filter's settings: the mount as (x, y, z, yaw) in float, the yaw's cosine and sine taken in double by
// the host C library, the thresholds squared in float (the node handle squares them in double, as InitParams does).
// The basis's third column is -0.0, a deliberate choice: Matrix3x3::setRotation of a yaw quaternion generally puts
// +0.0 there, but tf_apply adds z * m[i][2] before the translation, and a projected beam has z = +0, so with -0.0 that
// term is -0.0 and keeps the sign of an exactly-zero rotated sum.  Every beam then lands where c*x - s*y + lx and
// s*x + c*y + ly put it, bit for bit, as b2s_hector_scan_filter's conversion always has; with +0.0, a rotated sum of -0
// plus a -0.0 translation would come out +0.  Do not change it to match setRotation's basis.  Only a caller point with
// z < 0 or z = -0.0 (b2s_ros_hector_points) sees the term as +0.0: there an exactly-zero coordinate may be +0 where
// c*x - s*y + lx gives -0, which is tf's own arithmetic (Transform::operator*) on this basis.
inline HectorBeamFilter hector_scan_filter(const float laser_in_base[4], float scale_to_map, float min_dist, float max_dist,
                                           double use_max_scan_range, float z_min, float z_max) {
  HectorBeamFilter f;
  f.sqr_min = min_dist * min_dist;
  f.sqr_max = max_dist * max_dist;
  f.use_max_scan_range = use_max_scan_range;
  const double c = cos((double)laser_in_base[3]), s = sin((double)laser_in_base[3]);
  f.mount.m[0][0] = c; f.mount.m[0][1] = -s; f.mount.m[0][2] = -0.0;
  f.mount.m[1][0] = s; f.mount.m[1][1] = c; f.mount.m[1][2] = -0.0;
  f.mount.m[2][0] = 0.0; f.mount.m[2][1] = 0.0; f.mount.m[2][2] = 1.0;
  f.mount.o[0] = laser_in_base[0]; f.mount.o[1] = laser_in_base[1]; f.mount.o[2] = laser_in_base[2];
  f.z_min = z_min; f.z_max = z_max;
  f.scale_to_map = scale_to_map;
  return f;
}

// One processor's laser in the batched stream kernel's ingest (hector_slam.cu: HsIngest::lasers).  Scan i (a call-wide
// scan index) is the n_ranges floats at ranges + base + i * n_ranges.  Ranges are processor-major and ragged, so base
// is the processor's first float minus its first scan index times n_ranges: it may be negative, the sum is not.
struct HsLaser {
  HectorBeamFilter filter;
  long long base;
  int unit0;            // the first of its n_ranges unit vectors ([n][2] double) in the call's table
  int n_ranges;
  float range_min;
  double range_cutoff;  // projectLaser's cutoff (a negative one already replaced by range_max)
};

// The node handle's staging for its map publishes (hector_node.cu owns it, hs_node_run in hector_slam.cu fills it): a
// copy stream, two slots of level-0 payloads (one per node publishing before a part) on the device and page-locked on
// the host, and the per-scan record rows
struct HsNodeIo {
  Stream copy;
  Buf<int8_t> d_map[2];
  HostBuf<int8_t> h_map[2];  // a slot holds the payloads published before one part, back to back
  Event converted[2], copied[2];
  HostBuf<float> h_rows;  // [scans of the call][16], part-major: a part's rows are here once the next part's `copied` fired
};

// rosPointCloudToDataContainer (hector_slam.cc:331-358) on one laser-frame point: true if the node keeps it, with its
// DataContainer entry (base_link position in map-cell units) in (ox, oy).  laserTransform * Vector3(x, y, z) row by row
// (tf::Transform::operator*), the z window on that z minus the mount's z.
__host__ __device__ __forceinline__ bool hector_node_filter_point(const HectorBeamFilter &f, float x, float y, float z,
                                                                  float &ox, float &oy) {
  const float dist_sqr = x * x + y * y;
  if (!((dist_sqr > f.sqr_min) && (dist_sqr < f.sqr_max))) return false;
  if ((x < 0.0f) && (dist_sqr < 0.50f)) return false;  // behind the robot
  if ((double)dist_sqr > f.use_max_scan_range * f.use_max_scan_range) return false;
  const double v[3] = {(double)x, (double)y, (double)z};
  double b[3];
  tf_apply(f.mount, v, b);
  const float z_laser = (float)(b[2] - f.mount.o[2]);
  if (!(z_laser > f.z_min && z_laser < f.z_max)) return false;
  ox = (float)b[0] * f.scale_to_map;
  oy = (float)b[1] * f.scale_to_map;
  return true;
}

// projectLaser and the node's conversion on one beam
__host__ __device__ __forceinline__ bool hector_node_beam(const HectorBeamFilter &f, float range, double ux, double uy,
                                                          double cutoff, float range_min, float &ox, float &oy) {
  float x, y;
  if (!hector_project_beam(range, ux, uy, cutoff, range_min, x, y)) return false;
  return hector_node_filter_point(f, x, y, 0.0f, ox, oy);
}

// getUnitVectors_: cos / sin(angle_min + (double)i * angle_increment) in double by the host C library, the float32 message
// fields widened; interleaved [n][2].  angle_max only names laser_geometry's cache.
inline void hector_unit_vectors(float angle_min, float angle_increment, int n, double *out) {
  for (int i = 0; i < n; i++) {
    const double a = (double)angle_min + (double)i * (double)angle_increment;
    out[2 * i] = cos(a);
    out[2 * i + 1] = sin(a);
  }
}

// projectLaser's cutoff: a negative range_cutoff means the message's range_max
inline double hector_range_cutoff(double range_cutoff, float range_max) { return range_cutoff < 0.0 ? (double)range_max : range_cutoff; }

}  // namespace b2s
