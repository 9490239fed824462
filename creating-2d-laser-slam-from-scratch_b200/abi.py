"""ctypes mirrors of the plain-C structs in include/b200slam.h (layout must match field for field)."""
from __future__ import annotations

import ctypes as C

KT_PI_180 = 0.01745329251994329577  # Math.h:35

B2S_OK, B2S_ERR_BAD_PARAMS, B2S_ERR_OUT_OF_RANGE, B2S_ERR_NO_BEST_POSE = 0, 1, 2, 3
B2S_ERR_CUDA, B2S_ERR_NO_DEVICE, B2S_ERR_BAD_STATE, B2S_ERR_TOO_LARGE = 4, 5, 6, 7
STATUS_NAMES = {0: "OK", 1: "BAD_PARAMS", 2: "OUT_OF_RANGE", 3: "NO_BEST_POSE", 4: "CUDA", 5: "NO_DEVICE",
                6: "BAD_STATE", 7: "TOO_LARGE"}


class MatcherParams(C.Structure):
    """b2s_matcher_params.  Defaults are the reference's (Mapper.cpp:1569-1652)."""
    _fields_ = [("search_size", C.c_double), ("resolution", C.c_double), ("smear_deviation", C.c_double),
                ("range_threshold", C.c_double), ("distance_variance_penalty", C.c_double),
                ("angle_variance_penalty", C.c_double), ("fine_search_angle_offset", C.c_double),
                ("coarse_search_angle_offset", C.c_double), ("coarse_angle_resolution", C.c_double),
                ("minimum_angle_penalty", C.c_double), ("minimum_distance_penalty", C.c_double),
                ("use_response_expansion", C.c_int32), ("reserved", C.c_int32)]


def matcher_params(search_size=0.3, resolution=0.01, smear_deviation=0.03, range_threshold=12.0, **kw) -> MatcherParams:
    p = MatcherParams(search_size, resolution, smear_deviation, range_threshold,
                      0.3 * 0.3, (20 * KT_PI_180) ** 2, 0.2 * KT_PI_180, 20 * KT_PI_180, 2 * KT_PI_180,
                      0.9, 0.5, 0, 0)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class Laser(C.Structure):
    """b2s_laser."""
    _fields_ = [("n_readings", C.c_int32), ("reserved", C.c_int32), ("min_angle", C.c_double),
                ("angular_resolution", C.c_double), ("min_range", C.c_double), ("max_range", C.c_double),
                ("range_threshold", C.c_double), ("offset_pose", C.c_double * 3)]


def laser_from(l, n_readings=None) -> Laser:
    """From a synth.Laser-like object."""
    return Laser(l.n_readings if n_readings is None else n_readings, 0, l.min_angle, l.angular_resolution,
                 l.min_range, l.max_range, l.range_threshold, (C.c_double * 3)(*l.offset_pose))


class GridInfo(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("width", "height", "width_step", "data_size", "roi_x", "roi_y", "roi_w",
                                         "roi_h", "kernel_size", "search_side")]


class Search(C.Structure):
    _fields_ = [("offset_x", C.c_double), ("offset_y", C.c_double), ("res_x", C.c_double), ("res_y", C.c_double),
                ("angle_offset", C.c_double), ("angle_res", C.c_double), ("do_penalize", C.c_int32),
                ("fine", C.c_int32)]


class MatchResult(C.Structure):
    _fields_ = [("response", C.c_double), ("pose", C.c_double * 3), ("cov", C.c_double * 9),
                ("status", C.c_int32), ("tie_count", C.c_int32)]


class OccGridInfo(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("width_step", C.c_int32), ("data_size", C.c_int32),
                ("offset", C.c_double * 2), ("resolution", C.c_double), ("cell_visits", C.c_uint64)]


class IcpParams(C.Structure):
    """b2s_icp_params; defaults = lesson3/src/plicp_odometry.cc:72-185."""
    _fields_ = [("max_angular_correction_deg", C.c_double), ("max_linear_correction", C.c_double),
                ("epsilon_xy", C.c_double), ("epsilon_theta", C.c_double), ("max_correspondence_dist", C.c_double),
                ("outliers_maxPerc", C.c_double), ("outliers_adaptive_order", C.c_double),
                ("outliers_adaptive_mult", C.c_double), ("max_iterations", C.c_int32),
                ("use_point_to_line_distance", C.c_int32), ("outliers_remove_doubles", C.c_int32),
                ("reserved", C.c_int32)]


def icp_params(**kw) -> IcpParams:
    p = IcpParams(45.0, 1.0, 1e-6, 1e-6, 1.0, 0.90, 0.7, 2.0, 10, 1, 1, 0)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class IcpResult(C.Structure):
    _fields_ = [("x", C.c_double * 3), ("error", C.c_double), ("valid", C.c_int32), ("iterations", C.c_int32),
                ("nvalid", C.c_int32), ("reserved", C.c_int32)]


class PlicpOdomParams(C.Structure):
    """b2s_plicp_odom_params; defaults = lesson3/src/plicp_odometry.cc:64-67 and an identity laser mount."""
    _fields_ = [("icp", IcpParams), ("kf_dist_linear", C.c_double), ("kf_dist_angular", C.c_double),
                ("kf_scan_count", C.c_int32), ("reserved", C.c_int32), ("base_to_laser", C.c_double * 7)]


def plicp_odom_params(icp=None, base_to_laser=(0, 0, 0, 0, 0, 0, 1), **kw) -> PlicpOdomParams:
    import math
    p = PlicpOdomParams(icp if icp is not None else icp_params(), 0.1, 5.0 * (math.pi / 180.0), 10, 0,
                        (C.c_double * 7)(*base_to_laser))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class PlicpOdomLaser(C.Structure):
    """b2s_plicp_odom_laser: one recording's LaserScan fields (float32 angles, as the message carries them)."""
    _fields_ = [("n_beams", C.c_int32), ("angle_min", C.c_float), ("angle_increment", C.c_float),
                ("reserved", C.c_int32)]


class PlicpOdomStep(C.Structure):
    """b2s_plicp_odom_step."""
    _fields_ = [("position", C.c_double * 3), ("orientation", C.c_double * 4), ("linear", C.c_double * 3),
                ("angular", C.c_double * 3), ("first_guess", C.c_double * 3), ("icp", IcpResult),
                ("published", C.c_int32), ("keyframe", C.c_int32), ("reference_scan", C.c_int32),
                ("reserved", C.c_int32)]


class PlicpScanMatchStep(C.Structure):
    """b2s_plicp_scan_match_step."""
    _fields_ = [("icp", IcpResult), ("theta_deg", C.c_double), ("matched", C.c_int32), ("reserved", C.c_int32)]


# lesson3/src/scan_match_plicp.cc:38-157 (InitParams): the parameter-server names the node reads.  The first group maps
# onto b2s_icp_params; the second only speeds up the correspondence search or matters under a switch of the third
# group; the third selects CSM code paths the library does not build, so a non-zero value is refused.
_SCAN_MATCH_ICP = ("max_angular_correction_deg", "max_linear_correction", "max_iterations", "epsilon_xy",
                   "epsilon_theta", "max_correspondence_dist", "use_point_to_line_distance", "outliers_maxPerc",
                   "outliers_adaptive_order", "outliers_adaptive_mult", "outliers_remove_doubles")
_SCAN_MATCH_NO_EFFECT = ("sigma", "use_corr_tricks", "restart_threshold_mean_error", "restart_dt", "restart_dtheta",
                         "clustering_threshold", "orientation_neighbourhood", "do_alpha_test_thresholdDeg")
_SCAN_MATCH_REFUSED = ("restart", "do_alpha_test", "do_visibility_test", "do_compute_covariance", "debug_verify_tricks",
                       "use_ml_weights", "use_sigma_weights")


def plicp_scan_match_params(ros: dict | None = None) -> IcpParams:
    """ScanMatchPLICP::InitParams over a ROS parameter dict: absent keys keep the node's defaults (the same as
    icp_params()).  Switches of CSM code paths the library does not build (restart, do_alpha_test, ...) are refused
    with ValueError when non-zero, and names the node never reads with KeyError."""
    p = icp_params()
    for k, v in dict(ros or {}).items():
        if k in _SCAN_MATCH_ICP:
            setattr(p, k, int(v) if isinstance(getattr(p, k), int) else float(v))
        elif k in _SCAN_MATCH_REFUSED:
            if int(v) != 0:
                raise ValueError(f"{k} = {v}: this CSM switch is not built")
        elif k not in _SCAN_MATCH_NO_EFFECT:
            raise KeyError(f"{k} is not a parameter of the lesson3 scan-match node")
    return p


class PclIcpParams(C.Structure):
    """b2s_pcl_icp_params; defaults = a default-constructed pcl::IterativeClosestPoint (lesson2 scan_match_icp.h:49)."""
    _fields_ = [("max_iterations", C.c_int32), ("drop_invalid_points", C.c_int32),
                ("max_correspondence_distance", C.c_double), ("transformation_epsilon", C.c_double),
                ("euclidean_fitness_epsilon", C.c_double)]


def pcl_icp_params(**kw) -> PclIcpParams:
    import sys
    p = PclIcpParams(10, 0, sys.float_info.max ** 0.5, 0.0, -sys.float_info.max)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class PclIcpResult(C.Structure):
    _fields_ = [("x", C.c_float * 3), ("converged", C.c_int32), ("iterations", C.c_int32),
                ("n_correspondences", C.c_int32), ("fitness_score", C.c_double)]


def karto_round(v: float) -> float:
    """math::Round (Math.h:87-90)."""
    import math
    return math.floor(v + 0.5) if v >= 0.0 else math.ceil(v - 0.5)


def n_steps(off: float, res: float) -> int:
    """static_cast<kt_int32u>(math::Round(off * 2.0 / res) + 1) (Mapper.cpp:339-341)."""
    return int(karto_round(off * 2.0 / res) + 1)
