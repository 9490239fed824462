"""ctypes harness over the C ABI — K3 (lesson3): batched PL-ICP (sm_icp call site, plicp_odometry.cc:391) and the
odometry node around it (ScanMatchPLICP, plicp_odometry.cc:191-517) for B recordings at once."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .matcher import check, lib, f64, _d

_bound = False


def _bind():
    global _bound
    L = lib()
    if not _bound:
        dp = C.POINTER(C.c_double)
        L.b2s_plicp_match.argtypes = [C.POINTER(abi.IcpParams), C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double,
                                      dp, C.c_int, C.c_void_p, C.POINTER(abi.IcpResult)]
        L.b2s_plicp_odom_create.argtypes = [C.POINTER(abi.PlicpOdomParams), C.c_int, C.c_int, C.c_float, C.c_float,
                                            C.c_float, C.c_float, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
        L.b2s_plicp_odom_destroy.argtypes = [C.c_void_p]
        L.b2s_plicp_odom_destroy.restype = None
        L.b2s_plicp_odom_process.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                             C.POINTER(C.c_uint32), C.POINTER(abi.PlicpOdomStep)]
        L.b2s_plicp_odom_reset.argtypes = [C.c_void_p, C.c_int]
        _bound = True
    return L


def match(params: abi.IcpParams, ref_ranges, sens_ranges, theta, range_min, range_max, first_guess, device=0,
          stream=None):
    """-> (x[B,3], valid[B], iterations[B], nvalid[B], error[B])"""
    L = _bind()
    t = f64(theta)
    n = len(t)
    r, s = f64(ref_ranges).reshape(-1, n), f64(sens_ranges).reshape(-1, n)
    g = f64(first_guess).reshape(-1, 3)
    B = len(r)
    res = (abi.IcpResult * B)()
    check(L.b2s_plicp_match(C.byref(params), B, n, _d(r), _d(s), _d(t), range_min, range_max, _d(g), device,
                            C.c_void_p(stream) if stream else None, res))
    raw = np.frombuffer(res, dtype=np.dtype([("x", "<f8", 3), ("error", "<f8"), ("valid", "<i4"), ("iterations", "<i4"),
                                             ("nvalid", "<i4"), ("reserved", "<i4")]), count=B)
    return raw["x"].copy(), raw["valid"].copy(), raw["iterations"].copy(), raw["nvalid"].copy(), raw["error"].copy()


# one b2s_plicp_odom_step as a numpy record
STEP_DTYPE = np.dtype([("position", "<f8", 3), ("orientation", "<f8", 4), ("linear", "<f8", 3), ("angular", "<f8", 3),
                       ("first_guess", "<f8", 3), ("x", "<f8", 3), ("error", "<f8"), ("valid", "<i4"),
                       ("iterations", "<i4"), ("nvalid", "<i4"), ("icp_reserved", "<i4"), ("published", "<i4"),
                       ("keyframe", "<i4"), ("reference_scan", "<i4"), ("reserved", "<i4")])


class Odometry:
    """B ScanMatchPLICP nodes of one laser on the device (b2s_plicp_odom_*).  angle_min, angle_increment, range_min and
    range_max are the LaserScan's float32 fields."""

    def __init__(self, params: abi.PlicpOdomParams, batch, n_beams, angle_min, angle_increment, range_min, range_max,
                 device=0, stream=None):
        L = _bind()
        self._h = C.c_void_p()
        self.batch, self.n = int(batch), int(n_beams)
        check(L.b2s_plicp_odom_create(C.byref(params), self.batch, self.n, angle_min, angle_increment, range_min,
                                      range_max, device, C.c_void_p(stream) if stream else None, C.byref(self._h)))

    def process(self, recordings, stamps):
        """recordings: B arrays [S_b][n] float32 ranges (S_b = 0 leaves recording b untouched); stamps: B arrays
        [S_b][2] (sec, nsec).  -> list of B structured arrays of STEP_DTYPE, one row per scan."""
        counts = np.array([len(r) for r in recordings], np.int32)
        if len(counts) != self.batch or len(stamps) != self.batch or any(len(s) != c for s, c in zip(stamps, counts)):
            raise ValueError("one recording and one stamp per scan for every recording of the handle")
        total = int(counts.sum())
        rng = np.ascontiguousarray(np.concatenate([np.asarray(r, np.float32).reshape(-1, self.n) for r in recordings])
                                   if total else np.zeros((0, self.n), np.float32))
        stm = np.ascontiguousarray(np.concatenate([np.asarray(s, np.uint32).reshape(-1, 2) for s in stamps])
                                   if total else np.zeros((0, 2), np.uint32))
        out = (abi.PlicpOdomStep * max(total, 1))()
        check(_bind().b2s_plicp_odom_process(self._h, counts.ctypes.data_as(C.POINTER(C.c_int32)),
                                             rng.ctypes.data_as(C.POINTER(C.c_float)),
                                             stm.ctypes.data_as(C.POINTER(C.c_uint32)), out))
        raw = np.frombuffer(out, dtype=STEP_DTYPE, count=total).copy()
        return np.split(raw, np.cumsum(counts)[:-1])

    def reset(self, recording=-1):
        check(_bind().b2s_plicp_odom_reset(self._h, int(recording)))

    def close(self):
        if self._h:
            _bind().b2s_plicp_odom_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
