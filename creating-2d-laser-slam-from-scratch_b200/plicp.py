"""ctypes harness over the C ABI — K3 (lesson3): batched PL-ICP (sm_icp call site, plicp_odometry.cc:391), the
odometry node around it (ScanMatchPLICP, plicp_odometry.cc:191-517) and the scan-to-scan node (ScanMatchPLICP,
scan_match_plicp.cc:162-300), each for B recordings at once."""
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
        ip, fp = C.POINTER(C.c_int32), C.POINTER(C.c_float)
        L.b2s_plicp_scan_match_create.argtypes = [C.POINTER(abi.IcpParams), C.c_int, ip, fp, fp, C.c_int, C.c_void_p,
                                                  C.POINTER(C.c_void_p)]
        L.b2s_plicp_scan_match_destroy.argtypes = [C.c_void_p]
        L.b2s_plicp_scan_match_destroy.restype = None
        L.b2s_plicp_scan_match_process.argtypes = [C.c_void_p, ip, fp, fp, C.POINTER(abi.PlicpScanMatchStep)]
        L.b2s_plicp_scan_match_reset.argtypes = [C.c_void_p, C.c_int]
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


# one b2s_plicp_scan_match_step as a numpy record
SCAN_MATCH_STEP_DTYPE = np.dtype([("x", "<f8", 3), ("error", "<f8"), ("valid", "<i4"), ("iterations", "<i4"),
                                  ("nvalid", "<i4"), ("icp_reserved", "<i4"), ("theta_deg", "<f8"), ("matched", "<i4"),
                                  ("reserved", "<i4")])


class ScanMatch:
    """B lesson3 scan-to-scan ScanMatchPLICP nodes on the device (b2s_plicp_scan_match_*), one laser per recording:
    n_beams, angle_min and angle_increment are [B] (the LaserScans' float32 fields).  `params` is an abi.IcpParams,
    e.g. abi.plicp_scan_match_params(ros_params)."""

    def __init__(self, params: abi.IcpParams, n_beams, angle_min, angle_increment, device=0, stream=None):
        L = _bind()
        self._h = C.c_void_p()
        self.n = np.ascontiguousarray(n_beams, np.int32).reshape(-1)
        self.batch = len(self.n)
        amin = np.ascontiguousarray(angle_min, np.float32).reshape(-1)
        ainc = np.ascontiguousarray(angle_increment, np.float32).reshape(-1)
        if len(amin) != self.batch or len(ainc) != self.batch:
            raise ValueError("one beam count, angle_min and angle_increment per recording")
        check(L.b2s_plicp_scan_match_create(C.byref(params), self.batch, self.n.ctypes.data_as(C.POINTER(C.c_int32)),
                                            amin.ctypes.data_as(C.POINTER(C.c_float)),
                                            ainc.ctypes.data_as(C.POINTER(C.c_float)), device,
                                            C.c_void_p(stream) if stream else None, C.byref(self._h)))

    def process(self, recordings, range_limits):
        """recordings: B arrays [S_b][n_beams[b]] float32 ranges (S_b = 0 leaves recording b untouched);
        range_limits: B arrays [S_b][2] float32 (range_min, range_max of each scan).  -> list of B structured arrays
        of SCAN_MATCH_STEP_DTYPE, one row per scan."""
        if len(recordings) != self.batch or len(range_limits) != self.batch:
            raise ValueError("one recording and one range-limit array per recording of the handle")
        rec = [np.asarray(r, np.float32) for r in recordings]
        if any(r.size and (r.ndim != 2 or r.shape[1] != self.n[b]) for b, r in enumerate(rec)):
            raise ValueError("recording b is [S_b][n_beams[b]]")
        rec = [r.reshape(-1, self.n[b]) for b, r in enumerate(rec)]
        lim = [np.asarray(l, np.float32).reshape(-1, 2) for l in range_limits]
        counts = np.array([len(r) for r in rec], np.int32)
        if any(len(l) != c for l, c in zip(lim, counts)):
            raise ValueError("one (range_min, range_max) per scan")
        total = int(counts.sum())
        rng = np.ascontiguousarray(np.concatenate([r.reshape(-1) for r in rec]) if total else np.zeros(1, np.float32))
        lm = np.ascontiguousarray(np.concatenate(lim) if total else np.zeros((1, 2), np.float32))
        out = (abi.PlicpScanMatchStep * max(total, 1))()
        check(_bind().b2s_plicp_scan_match_process(self._h, counts.ctypes.data_as(C.POINTER(C.c_int32)),
                                                   rng.ctypes.data_as(C.POINTER(C.c_float)),
                                                   lm.ctypes.data_as(C.POINTER(C.c_float)), out))
        raw = np.frombuffer(out, dtype=SCAN_MATCH_STEP_DTYPE, count=total).copy()
        return np.split(raw, np.cumsum(counts)[:-1])

    def reset(self, recording=-1):
        check(_bind().b2s_plicp_scan_match_reset(self._h, int(recording)))

    def close(self):
        if self._h:
            _bind().b2s_plicp_scan_match_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
