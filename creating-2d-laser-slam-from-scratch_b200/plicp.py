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
        L.b2s_plicp_odom_create_fleet.argtypes = [C.c_int, C.POINTER(abi.PlicpOdomParams), C.POINTER(abi.PlicpOdomLaser),
                                                  C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
        L.b2s_plicp_odom_process_fleet.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                                   C.POINTER(C.c_float), C.POINTER(C.c_uint32),
                                                   C.POINTER(abi.PlicpOdomStep)]
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
    """B ScanMatchPLICP nodes on the device (b2s_plicp_odom_*).  The constructor makes B nodes of one laser, one
    parameter set and fixed range fields (b2s_plicp_odom_create); Odometry.fleet gives every recording its own
    parameters and laser, the range fields coming with every scan.  Angles and range fields are the LaserScan's
    float32 fields."""

    def __init__(self, params: abi.PlicpOdomParams, batch, n_beams, angle_min, angle_increment, range_min, range_max,
                 device=0, stream=None):
        L = _bind()
        self._h = C.c_void_p()
        self.batch, self.n = int(batch), int(n_beams)
        self.n_beams = np.full(max(self.batch, 0), self.n, np.int32)
        self.has_fields = True
        check(L.b2s_plicp_odom_create(C.byref(params), self.batch, int(n_beams), angle_min, angle_increment, range_min,
                                      range_max, device, C.c_void_p(stream) if stream else None, C.byref(self._h)))

    @classmethod
    def fleet(cls, params_list, n_beams, angle_min, angle_increment, device=0, stream=None):
        """One node per recording: params_list [B] of abi.PlicpOdomParams, n_beams / angle_min / angle_increment [B]
        (b2s_plicp_odom_create_fleet).  process() then needs each scan's range fields."""
        L = _bind()
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.n = self.n_beams = np.ascontiguousarray(n_beams, np.int32).reshape(-1)
        self.batch = len(self.n_beams)
        self.has_fields = False
        amin = np.asarray(angle_min, np.float32).reshape(-1)
        ainc = np.asarray(angle_increment, np.float32).reshape(-1)
        params_list = list(params_list)
        if len(params_list) != self.batch or len(amin) != self.batch or len(ainc) != self.batch:
            raise ValueError("one parameter set, beam count, angle_min and angle_increment per recording")
        P = (abi.PlicpOdomParams * max(self.batch, 1))(*params_list)
        lasers = (abi.PlicpOdomLaser * max(self.batch, 1))(
            *[abi.PlicpOdomLaser(int(n), float(a), float(i), 0) for n, a, i in zip(self.n, amin, ainc)])
        check(L.b2s_plicp_odom_create_fleet(self.batch, P, lasers, device, C.c_void_p(stream) if stream else None,
                                            C.byref(self._h)))
        return self

    def process(self, recordings, stamps, range_limits=None):
        """recordings: B arrays [S_b][n_beams[b]] float32 ranges (S_b = 0 leaves recording b untouched); stamps: B
        arrays [S_b][2] (sec, nsec); range_limits: B arrays [S_b][2] float32 (range_min, range_max of each scan),
        required on a fleet handle, else the create-time fields.  -> list of B structured arrays of STEP_DTYPE, one row
        per scan."""
        if len(recordings) != self.batch or len(stamps) != self.batch or \
                (range_limits is not None and len(range_limits) != self.batch):
            raise ValueError("one recording, stamp array and range-limit array per recording of the handle")
        if range_limits is None and not self.has_fields:
            raise ValueError("a fleet handle needs each scan's (range_min, range_max)")
        rec = [np.asarray(r, np.float32) for r in recordings]
        if not self.has_fields and any(r.size and (r.ndim != 2 or r.shape[1] != self.n_beams[b])
                                       for b, r in enumerate(rec)):
            raise ValueError("recording b is [S_b][n_beams[b]]")
        rec = [r.reshape(-1, self.n_beams[b]) for b, r in enumerate(rec)]
        counts = np.array([len(r) for r in rec], np.int32)
        stm = [np.asarray(s, np.uint32).reshape(-1, 2) for s in stamps]
        if any(len(s) != c for s, c in zip(stm, counts)):
            raise ValueError("one stamp per scan")
        total = int(counts.sum())
        rng = np.ascontiguousarray(np.concatenate([r.reshape(-1) for r in rec]) if total else np.zeros(1, np.float32))
        st = np.ascontiguousarray(np.concatenate(stm) if total else np.zeros((1, 2), np.uint32))
        out = (abi.PlicpOdomStep * max(total, 1))()
        ip, fp, up = C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_uint32)
        if range_limits is None:
            check(_bind().b2s_plicp_odom_process(self._h, counts.ctypes.data_as(ip), rng.ctypes.data_as(fp),
                                                 st.ctypes.data_as(up), out))
        else:
            lim = [np.asarray(l, np.float32).reshape(-1, 2) for l in range_limits]
            if any(len(l) != c for l, c in zip(lim, counts)):
                raise ValueError("one (range_min, range_max) per scan")
            lm = np.ascontiguousarray(np.concatenate(lim) if total else np.zeros((1, 2), np.float32))
            check(_bind().b2s_plicp_odom_process_fleet(self._h, counts.ctypes.data_as(ip), rng.ctypes.data_as(fp),
                                                       lm.ctypes.data_as(fp), st.ctypes.data_as(up), out))
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
