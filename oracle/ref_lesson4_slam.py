"""TEST INFRASTRUCTURE — ctypes binding of oracle/_ref/liblesson4_slam_ref.so: lesson4's UNMODIFIED Hector SLAM node,
reference/lesson4/src/hector_mapping/hector_slam.cc, compiled where it lies against the stand-ins under
oracle/shim_lesson4_slam/, oracle/shim_lesson6/ and oracle/shim/ by oracle/ref_lesson4_slam.cpp (its own translation
unit), built by oracle/recipes.py from a checkout of the original project; where it is absent the tests replay its
recorded answers (tests/reference_record.py).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import recipes

_NAME = "_ref/liblesson4_slam_ref.so"
_lib = None


def available() -> bool:
    return recipes.available(_NAME)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(recipes.path(_NAME))
        vp = C.c_void_p
        L.ref_l4s_clear_params.argtypes = []
        L.ref_l4s_clear_params.restype = None
        L.ref_l4s_param.argtypes = [C.c_char_p, C.c_double]
        L.ref_l4s_param.restype = None
        L.ref_l4s_new.argtypes = [vp]
        L.ref_l4s_new.restype = None
        L.ref_l4s_scan.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
        L.ref_l4s_publish.argtypes = [vp, vp, vp, C.c_long, vp]
        _lib = L
    return _lib


def run(params: dict, geometry, mount, ranges, stamps, schedule):
    """A fresh node with the parameter-server values `params` (InitParams' names, numbers) and the laser mount over one
    recording.  geometry = (angle_min, angle_increment, range_min, range_max) float32, ranges [S][n] float32, stamps
    [S][2].  schedule.before(stamp) names the tick of the map published before each scan, or None (the library's
    schedule: the node's own runs on a thread).  -> dict(pose, pose_msg, cov, tf [S][2][7], n_points, maps [dict])."""
    L = lib()
    L.ref_l4s_clear_params()
    for k, v in params.items():
        L.ref_l4s_param(k.encode(), float(v))
    m = np.ascontiguousarray(mount, np.float64)
    L.ref_l4s_new(m.ctypes.data)
    f = np.ascontiguousarray(geometry, np.float32)
    r = np.ascontiguousarray(ranges, np.float32)
    st = np.ascontiguousarray(stamps, np.uint32)
    S = len(r)
    out = dict(pose=np.zeros((S, 3), np.float32), pose_msg=np.zeros((S, 7)), cov=np.zeros((S, 36)),
               tf=np.zeros((S, 2, 7)), n_points=np.zeros(S, np.int32), maps=[])
    payload = None
    for i in range(S):
        tick = schedule.before(st[i])
        if tick is not None:
            t = np.array(tick, np.uint32)
            info = np.zeros(5)
            rebuilt = C.c_int32(0)
            if payload is None:
                payload = np.zeros(1 << 26, np.int8)
            rc = L.ref_l4s_publish(t.ctypes.data, info.ctypes.data, payload.ctypes.data, payload.size, C.addressof(rebuilt))
            assert rc == 0, f"publishMap before scan {i}: {rc}"
            w, h = int(info[3]), int(info[4])
            out["maps"].append(dict(scan_index=i, stamp=tuple(int(v) for v in tick),
                                    info=dict(origin_x=float(info[0]), origin_y=float(info[1]), resolution=float(info[2]),
                                              width=w, height=h),
                                    payload=payload[:w * h].reshape(h, w).copy(), rebuilt=bool(rebuilt.value)))
        n = C.c_int32(0)
        rc = L.ref_l4s_scan(f.ctypes.data, r.shape[1], r[i].ctypes.data, st[i].ctypes.data, out["pose"][i].ctypes.data,
                            out["pose_msg"][i].ctypes.data, out["cov"][i].ctypes.data, out["tf"][i].ctypes.data,
                            C.addressof(n))
        assert rc == 0, f"scanCallback of scan {i} did not publish its odometry and transforms"
        out["n_points"][i] = n.value
    return out
