"""Test recordings for lesson3's scan-to-scan node (ScanMatchPLICP, scan_match_plicp.cc:162-300) and the helpers every
scan-match test shares: the C restatement (orc_plicp_scan_match in oracle/plicp_scan_match_oracle.c), the unmodified
node's answers (live where oracle/_ref/ is built, replayed from tests/golden/reference/ elsewhere), and packing a run
into one array.

A recording is a dict: ranges [S][n] float32, limits [S][2] float32 (each message's range_min, range_max), the float32
angle_min and angle_increment of its laser, and the node's parameter-server values.  The scans are synthetic rooms
(synth.py), seeded."""
from __future__ import annotations

import importlib
import math

import numpy as np

import plicp_odometry_cases as oc

synth = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.synth")
abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")

HOKUYO = (np.float32(oc.FIELDS[0]), np.float32(oc.FIELDS[1]))
LIMITS = (np.float32(oc.FIELDS[2]), np.float32(oc.FIELDS[3]))


def recording(ranges, limits=None, laser=HOKUYO, params=None):
    r = np.ascontiguousarray(ranges, np.float32)
    lm = np.tile(np.array(LIMITS, np.float32), (len(r), 1)) if limits is None else np.asarray(limits, np.float32)
    return dict(ranges=r, limits=np.ascontiguousarray(lm.reshape(len(r), 2)), angle_min=np.float32(laser[0]),
                angle_increment=np.float32(laser[1]), params=dict(params or {}))


def drive(seed, steps, n=1081, laser=HOKUYO, sigma=0.005, start=(0.0, 0.0, 0.0)):
    """Ranges [len(steps) + 1][n] of a laser driven through a room: steps = (forward, left, turn in rad) before each scan
    after the first."""
    rng = np.random.default_rng(seed)
    world = synth.make_world(seed)
    lz = synth.Laser(n_readings=n, min_angle=float(laser[0]), angular_resolution=float(laser[1]))
    pose = np.array(start, np.float64)
    out = []
    for k in range(len(steps) + 1):
        if k:
            f, l, t = steps[k - 1]
            c, s = math.cos(pose[2]), math.sin(pose[2])
            pose = pose + np.array([c * f - s * l, s * f + c * l, t])
        out.append(synth.cast_scan(world, pose, lz, rng, sigma))
    return np.array(out).astype(np.float32)


def _edges():
    """Readings exactly at the float range_min / range_max (invalid), one float step inside them (valid), NaN, +-inf
    and 0, on every scan at different beams."""
    r = drive(31, [(0.02, 0.0, math.radians(0.5))] * 7)
    lo, hi = LIMITS
    for k in range(len(r)):
        b = 40 + 97 * k
        r[k, b:b + 5] = lo
        r[k, b + 5:b + 8] = np.nextafter(lo, np.float32(np.inf))
        r[k, b + 8:b + 12] = hi
        r[k, b + 12:b + 15] = np.nextafter(hi, np.float32(0))
        r[k, b + 15:b + 19] = np.nan
        r[k, b + 19:b + 22] = np.inf
        r[k, b + 22:b + 24] = -np.inf
        r[k, b + 24:b + 30] = 0.0
    return recording(r)


def _limits_change():
    """The range fields narrow and widen from scan to scan, so each pair mixes two windows."""
    r = drive(32, [(0.02, 0.01, math.radians(0.7))] * 11)
    lim = [(0.1, 30.0), (0.5, 6.0), (0.1, 30.0), (2.0, 4.5), (0.05, 40.0), (0.05, 40.0), (1.0, 8.0), (3.0, 5.0),
           (0.1, 30.0), (0.0, np.inf), (-np.inf, np.inf), (0.1, 30.0)]
    return recording(r, np.array(lim, np.float32))


def _streams():
    d = math.radians
    out = {}
    for name, st in oc.STREAMS.items():  # the odometry node's recordings, its ICP parameters only
        icp = {k: v for k, v in st["params"].items() if hasattr(abi.IcpParams, k)}
        out["odom_" + name] = recording(st["ranges"], params=icp)
    r2 = drive(33, [(0.03, 0.0, d(1.0))] * 5)
    out.update({
        "edges": _edges(),
        "limits_change": _limits_change(),
        "one_scan": recording(r2[:1]),
        "two_scans": recording(r2[:2]),
        "identical": recording(np.repeat(drive(34, [], sigma=0.0), 4, 0)),
        "beyond_max_angular": recording(drive(35, [(0.0, 0.0, d(90.0))] * 6),
                                        params=dict(max_angular_correction_deg=5.0, max_correspondence_dist=0.05)),
        "one_iteration": recording(drive(36, [(0.03, 0.0, d(1.0))] * 6), params=dict(max_iterations=1)),
        "point_to_point": recording(drive(37, [(0.03, 0.01, d(1.0))] * 6), params=dict(use_point_to_line_distance=0)),
        "keep_doubles": recording(drive(38, [(0.03, 0.0, d(-1.0))] * 6), params=dict(outliers_remove_doubles=0)),
        "full_circle": recording(drive(39, [(0.03, 0.0, d(2.0))] * 6, n=720,
                                       laser=(np.float32(-math.pi), np.float32(2 * math.pi / 720))),
                                 laser=(np.float32(-math.pi), np.float32(2 * math.pi / 720))),
        "no_effect_params": recording(drive(40, [(0.02, 0.0, d(1.0))] * 5),
                                      params=dict(sigma=0.05, use_corr_tricks=0, clustering_threshold=0.5,
                                                  orientation_neighbourhood=5, restart=0, do_alpha_test=0)),
    })
    return out


STREAMS = _streams()
REFUSED = {"restart": 1, "do_alpha_test": 1, "do_visibility_test": 1, "do_compute_covariance": 1, "use_ml_weights": 1,
           "use_sigma_weights": 1, "debug_verify_tricks": 1}


def icp_params(rec):
    """b2s_icp_params of a recording: the node's defaults overridden by its parameter-server values."""
    return abi.plicp_scan_match_params(rec["params"])


def restate(rec) -> np.ndarray:
    """orc_plicp_scan_match (the C restatement) over a recording -> structured array of SCAN_MATCH_STEP_DTYPE."""
    from oracle import plicp_scan_match_port
    return plicp_scan_match_port.scan_match(icp_params(rec), rec["angle_min"], rec["angle_increment"], rec["ranges"],
                                            rec["limits"])


FLOAT_FIELDS = ("x", "error", "theta_deg")
INT_FIELDS = ("valid", "iterations", "nvalid", "matched")


def pack(steps) -> np.ndarray:
    """[S][9] float64: every field of a run (integers widened exactly)."""
    cols = [np.asarray(steps[f], np.float64).reshape(len(steps), -1) for f in FLOAT_FIELDS + INT_FIELDS]
    return np.ascontiguousarray(np.concatenate(cols, 1))


def _inputs(rec):
    return (rec["ranges"], rec["limits"], float(rec["angle_min"]), float(rec["angle_increment"]),
            sorted(rec["params"].items()))


def node_answers(live):
    """{recording name: pack(node run)} from the unmodified node (oracle/ref_lesson3_scan_match.cpp), live or
    replayed; "refused:<switch>" -> whether the node threw on a two-scan recording with that switch set to 1."""
    from reference_record import Recording
    rec = Recording("test_plicp_scan_match_reference__node_streams", live)
    out = {}
    for name, st in STREAMS.items():
        def run(st=st):
            from oracle import ref_lesson3_scan_match
            return pack(ref_lesson3_scan_match.run(st["params"], st["angle_min"], st["angle_increment"], st["ranges"],
                                                   st["limits"]))
        out[name] = rec.value(name, run, inputs=_inputs(st))
    two = STREAMS["two_scans"]
    for k, v in sorted(REFUSED.items()):
        def threw(k=k, v=v):
            from oracle import ref_lesson3_scan_match
            try:
                ref_lesson3_scan_match.run({k: v}, two["angle_min"], two["angle_increment"], two["ranges"],
                                           two["limits"])
            except RuntimeError:
                return True
            return False
        out["refused:" + k] = rec.value("refused:" + k, threw, inputs=_inputs(two) + (k, v))
    rec.save()
    return out
