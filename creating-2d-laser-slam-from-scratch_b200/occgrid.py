"""ctypes harness over the C ABI — K2c, karto::OccupancyGrid::CreateFromScans (Karto.h:5659-5673)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from .matcher import check, lib, f64, _d

_bound = False


def _bind():
    global _bound
    L = lib()
    if _bound:
        return L
    vp = C.c_void_p
    L.b2s_occ_grid_create_from_scans.argtypes = [C.POINTER(abi.Laser), C.c_int, C.POINTER(C.c_double),
                                                 C.POINTER(C.c_double), C.c_double, C.c_int, vp, C.POINTER(vp)]
    dp, u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
    L.b2s_occ_grid_scans_bbox.argtypes = [C.POINTER(abi.Laser), C.c_int, dp, dp, C.c_int, vp, dp]
    L.b2s_occ_grid_create_shard.argtypes = [C.POINTER(abi.Laser), C.c_int, dp, dp, C.c_double, dp, C.c_int, vp,
                                            C.POINTER(vp)]
    L.b2s_occ_grid_device_counters.argtypes = [vp, C.POINTER(u32p), C.POINTER(u32p)]
    L.b2s_occ_grid_set_counters.argtypes = [vp, u32p, u32p]
    L.b2s_occ_grid_update.argtypes = [vp]
    L.b2s_occ_grid_info_get.argtypes = [vp, C.POINTER(abi.OccGridInfo)]
    L.b2s_occ_grid_copy.argtypes = [vp, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.b2s_occ_grid_copy_ros.argtypes = [vp, C.POINTER(C.c_int8)]
    L.b2s_occ_grid_last_timing.argtypes = [vp, C.POINTER(C.c_double)]
    L.b2s_occ_grid_destroy.argtypes = [vp]
    L.b2s_occ_grid_destroy.restype = None
    _bound = True
    return L


class _DeviceArray:
    """A device pointer of the library dressed with __cuda_array_interface__, so torch.as_tensor() can alias it (no
    copy) for an in-place NCCL all-reduce.  uint32 counters are exposed as int32: a sum of them has the same bits."""

    def __init__(self, ptr: int, n: int, owner):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}
        self.owner = owner  # keeps the grid handle alive


def scans_bbox(laser: abi.Laser, ranges, poses, device: int = 0, stream=None) -> np.ndarray:
    """BoundingBox2 {min x, min y, max x, max y} of a scan shard (Karto.h:5810-5814)"""
    L = _bind()
    p = f64(poses).reshape(-1, 3)
    r = f64(ranges).reshape(len(p), laser.n_readings)
    out = np.zeros(4)
    check(L.b2s_occ_grid_scans_bbox(C.byref(laser), len(p), _d(r), _d(p), device,
                                    C.c_void_p(stream) if stream else None, _d(out)))
    return out


class OccupancyGrid:
    """Stand-in for karto::OccupancyGrid* as returned by CreateFromScans.  With `bbox` the scans are one shard of a
    larger list and the grid is dimensioned by that (global) box; see b2s_occ_grid_create_shard."""

    def __init__(self, laser: abi.Laser, ranges, poses, resolution: float, device: int = 0, stream=None, bbox=None):
        self.L = _bind()
        p = f64(poses).reshape(-1, 3)
        r = f64(ranges).reshape(len(p), laser.n_readings)
        self.h = C.c_void_p()
        st = C.c_void_p(stream) if stream else None
        if bbox is None:
            check(self.L.b2s_occ_grid_create_from_scans(C.byref(laser), len(p), _d(r), _d(p), resolution, device, st,
                                                        C.byref(self.h)))
        else:
            check(self.L.b2s_occ_grid_create_shard(C.byref(laser), len(p), _d(r), _d(p), resolution, _d(f64(bbox)),
                                                   device, st, C.byref(self.h)))
        self.info = abi.OccGridInfo()
        if self.h.value:
            check(self.L.b2s_occ_grid_info_get(self.h, C.byref(self.info)))

    @property
    def is_null(self):
        return not self.h.value

    def arrays(self):
        i = self.info
        n = i.data_size
        cells, pas, hit = np.zeros(n, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        check(self.L.b2s_occ_grid_copy(self.h, cells.ctypes.data_as(C.POINTER(C.c_uint8)),
                                       pas.ctypes.data_as(C.POINTER(C.c_uint32)),
                                       hit.ctypes.data_as(C.POINTER(C.c_uint32))))
        sh = (i.height, i.width_step)
        return dict(width=i.width, height=i.height, width_step=i.width_step, offset=np.array(i.offset[:]),
                    cell_visits=int(i.cell_visits), cells=cells.reshape(sh), passes=pas.reshape(sh),
                    hits=hit.reshape(sh))

    def device_counters(self):
        """-> (pass, hit) as objects torch.as_tensor() aliases on the device (int32 view of the uint32 counters)"""
        dp_, dh_ = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
        check(self.L.b2s_occ_grid_device_counters(self.h, C.byref(dp_), C.byref(dh_)))
        n = self.info.data_size
        return (_DeviceArray(C.cast(dp_, C.c_void_p).value or 0, n, self),
                _DeviceArray(C.cast(dh_, C.c_void_p).value or 0, n, self))

    def allreduce_counters(self, nccl_comm):
        """b2s_occ_grid_allreduce_counters: both counter planes summed over the ranks in place by the library (NCCL)."""
        self.L.b2s_occ_grid_allreduce_counters.argtypes = [C.c_void_p, C.c_void_p]
        check(self.L.b2s_occ_grid_allreduce_counters(self.h, nccl_comm.comm))

    def set_counters(self, passes, hits):
        pa = np.ascontiguousarray(passes, np.uint32).reshape(-1)
        hi = np.ascontiguousarray(hits, np.uint32).reshape(-1)
        assert len(pa) == len(hi) == self.info.data_size
        check(self.L.b2s_occ_grid_set_counters(self.h, pa.ctypes.data_as(C.POINTER(C.c_uint32)),
                                               hi.ctypes.data_as(C.POINTER(C.c_uint32))))

    def update(self):
        """OccupancyGrid::Update (Karto.h:5953-5968): re-threshold the cells from the counters"""
        check(self.L.b2s_occ_grid_update(self.h))

    def ros_map(self):
        out = np.zeros((self.info.height, self.info.width), dtype=np.int8)
        check(self.L.b2s_occ_grid_copy_ros(self.h, out.ctypes.data_as(C.POINTER(C.c_int8))))
        return out

    def last_timing(self):
        out = np.zeros(2)
        check(self.L.b2s_occ_grid_last_timing(self.h, _d(out)))
        return dict(raytrace_ms=out[0], threshold_ms=out[1])

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.b2s_occ_grid_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


BATCH_GRID_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.POINTER(abi.OccGridInfo), C.POINTER(C.c_int8))


def create_from_scans_batch(laser: abi.Laser, ranges_list, poses_list, resolutions, device: int = 0):
    """b2s_occ_grid_create_from_scans_batch: grid g over ranges_list[g] [S_g][n] (float32) at poses_list[g] [S_g][3]
    with resolutions[g], every grid in one batched build.  -> one (info dict, payload [h][w] int8) per grid, None for a
    grid without scans."""
    L = _bind()
    L.b2s_occ_grid_create_from_scans_batch.argtypes = [C.POINTER(abi.Laser), C.c_int, C.POINTER(C.c_int32),
                                                       C.POINTER(C.c_float), C.POINTER(C.c_double),
                                                       C.POINTER(C.c_double), C.c_int, BATCH_GRID_FN, C.c_void_p]
    G = len(ranges_list)
    counts = np.array([len(r) for r in ranges_list], np.int32)
    n = laser.n_readings
    r = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float32).reshape(-1, n) for x in ranges_list])
                             if counts.sum() else np.zeros((0, n), np.float32))
    p = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64).reshape(-1, 3) for x in poses_list])
                             if counts.sum() else np.zeros((0, 3)))
    res = np.ascontiguousarray(resolutions, np.float64)
    out = [None] * G

    def cb(user, g, info_p, payload_p):
        i = info_p.contents
        info = dict(width=i.width, height=i.height, width_step=i.width_step, data_size=i.data_size,
                    offset=np.array(i.offset[:]), resolution=i.resolution, cell_visits=int(i.cell_visits))
        out[g] = (info, np.ctypeslib.as_array(payload_p, shape=(i.height * i.width,)).reshape(i.height, i.width).copy()
                  if i.height * i.width else np.zeros((i.height, i.width), np.int8))

    fn = BATCH_GRID_FN(cb)
    check(L.b2s_occ_grid_create_from_scans_batch(C.byref(laser), G, counts.ctypes.data_as(C.POINTER(C.c_int32)),
                                                 r.ctypes.data_as(C.POINTER(C.c_float)), _d(p), _d(res), device, fn,
                                                 None))
    return out
