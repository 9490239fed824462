"""Seeded LaserScan recordings and node parameters for lesson4's make-map nodes (gmapping.cc, hector_mapping.cc), shared
by the CPU test against the unmodified nodes and the GPU test against the restatement."""
from __future__ import annotations

import importlib

import numpy as np

node_maps = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.node_maps")

# a 270-degree laser of 1081 beams (the lesson bags' geometry), float32 fields as the message carries them
N = 1081
FIELDS = (np.float32(-2.35619449), np.float32(np.radians(0.25)), np.float32(0.1), np.float32(30.0))


def _box(half, n, shift=(0.0, 0.0), angle_min=FIELDS[0], inc=FIELDS[1]):
    """Ranges from the origin to the walls of the axis-aligned box [-hx, hx] x [-hy, hy] shifted by `shift`."""
    a = angle_min.astype(np.float64) + np.arange(n) * np.float64(inc)
    c, s = np.cos(a), np.sin(a)
    with np.errstate(divide="ignore"):
        tx = np.where(c > 0, (half[0] + shift[0]) / c, np.where(c < 0, (-half[0] + shift[0]) / c, np.inf))
        ty = np.where(s > 0, (half[1] + shift[1]) / s, np.where(s < 0, (-half[1] + shift[1]) / s, np.inf))
    return np.minimum(tx, ty)


def recording(seed, scans, half, sigma=0.01, dropouts=0.02, n=N, shift_step=(0.02, 0.01)):
    """`scans` noisy scans of a box room, the robot drifting by shift_step per scan; a `dropouts` share of each scan's
    beams is NaN, inf or 0 (a third each)."""
    rng = np.random.default_rng(seed)
    out = np.zeros((scans, n), np.float32)
    for k in range(scans):
        r = _box(half, n, (shift_step[0] * k, shift_step[1] * k)) + rng.normal(0, sigma, n)
        drop = rng.random(n) < dropouts
        kind = rng.integers(0, 3, n)
        r = r.astype(np.float32)
        r[drop & (kind == 0)] = np.nan
        r[drop & (kind == 1)] = np.inf
        r[drop & (kind == 2)] = 0.0
        out[k] = r
    return out


def edge_scan(max_range=30 - 0.01, max_use=25.0, range_min=FIELDS[2], range_max=FIELDS[3]):
    """One room scan whose beams sit on every filter edge of both nodes, each with its float neighbours."""
    r = recording(5, 1, (7.0, 5.0), dropouts=0.0)[0]
    lim = np.float32(range_max) - np.float32(0.1)  # hector_mapping.cc:150
    edges = []
    for v in (np.float32(max_range), np.float32(max_use), np.float32(range_min), lim, np.float32(max_use) * 0.5):
        edges += [np.nextafter(v, np.float32(-np.inf)), v, np.nextafter(v, np.float32(np.inf))]
    edges = np.array(edges, np.float32)
    idx = np.linspace(10, N - 10, len(edges) * 4).astype(int)
    r[idx] = np.tile(edges, 4)
    return r[None]


def _ros(params):
    """The node parameter names of a node_maps params structure (gmapping.cc:46-62 / hector_mapping.cc:46-55)."""
    names = {"max_range": "maxRange", "max_use_range": "maxUrange", "xmin": "xmin", "ymin": "ymin", "xmax": "xmax",
             "ymax": "ymax", "delta": "delta", "occ_thresh": "occ_thresh"}
    return {names[k]: float(getattr(params, k)) for k, _ in params._fields_ if k in names}


def gmapping_cases():
    """name -> (params, fields, ranges)"""
    P = node_maps.gmapping_params
    room, hall = recording(1, 3, (6.0, 4.0)), recording(2, 3, (35.0, 1.5))
    far = recording(6, 2, (60.0, 2.0), dropouts=0.0)
    # scans 0 and 1 stay inside a +-5 m map, scan 2 sees walls 6 m away: the node asserts on scan 2
    leaves = np.concatenate([recording(3, 2, (3.0, 2.0)), recording(4, 2, (6.0, 4.0))])
    return {
        "room_defaults": (P(), FIELDS, room),
        "hall_defaults": (P(), FIELDS, hall),
        "edges_defaults": (P(), FIELDS, edge_scan()),
        "exact_delta": (P(delta=0.0625), FIELDS, room),          # 80 / 0.0625 = 1280 in float and in double
        "small_storage": (P(xmin=-25.0, ymin=-25.0, xmax=25.0, ymax=25.0), FIELDS, room),  # payload 999, storage 992
        "asymmetric": (P(xmin=-12.0, ymin=-30.0, xmax=44.0, ymax=9.0, occ_thresh=0.4), FIELDS, hall[:, ::-1].copy()),
        "far_walls": (P(max_range=80.0, max_use_range=50.0, xmin=-64.0, ymin=-64.0, xmax=64.0, ymax=64.0),
                      FIELDS, far),
        "leaves_map": (P(xmin=-5.0, ymin=-5.0, xmax=5.0, ymax=5.0), FIELDS, leaves),
    }


def hector_cases():
    """name -> (params, fields, ranges)"""
    P = node_maps.hector_params
    room, hall = recording(1, 3, (6.0, 4.0)), recording(2, 3, (35.0, 1.5))
    far_fields = FIELDS[:3] + (np.float32(100.0),)
    return {
        "room_defaults": (P(), FIELDS, room),
        "hall_defaults": (P(), FIELDS, hall),
        "edges_defaults": (P(), FIELDS, edge_scan()),
        "exact_delta": (P(delta=0.0625), FIELDS, room),
        "small_map": (P(xmin=-25.0, ymin=-25.0, xmax=25.0, ymax=25.0), FIELDS, room),
        # beams up to 60 m end outside the 1599 x 1599 map (cell 800 + 1200): their lines are not drawn
        "beyond_map": (P(), far_fields, recording(6, 2, (60.0, 2.0), dropouts=0.0)),
        # the begin cell (800, 800) outside a 700-cell map: nothing is drawn
        "begin_outside": (P(xmin=-17.5, ymin=-17.5, xmax=17.5, ymax=17.5), FIELDS, room[:1]),
    }


def ros_params(params) -> dict:
    return _ros(params)
