"""Device memory that an entry point takes for the length of one call goes back, on success and on error: the default
memory pool's CU_MEMPOOL_ATTR_USED_MEM_CURRENT is the same before and after each call.  The library links cudart
statically, so the pool is read through the driver API."""
import ctypes as C

import numpy as np
import pytest

import deskew_cases as dc

pytestmark = pytest.mark.gpu

CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7


class _DefaultPool:
    def __init__(self, device=0):
        self.cu = C.CDLL("libcuda.so.1")
        assert self.cu.cuInit(0) == 0
        dev = C.c_int()
        assert self.cu.cuDeviceGet(C.byref(dev), device) == 0
        self.pool = C.c_void_p()
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def used(self):
        assert self.cu.cuCtxSynchronize() == 0  # stream-ordered frees take effect in stream order
        v = C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(v)) == 0
        return v.value


def _scans(pkg, n=6):
    laser = pkg.synth.Laser()
    _, poses, ranges = pkg.synth.make_trajectory(5, n, laser, step_xy=0.1, step_th_deg=3)
    return laser, poses, ranges


def occgrid_too_large(pkg):
    O, M, abi = pkg.load("occgrid"), pkg.load("matcher"), pkg.abi
    laser, poses, ranges = _scans(pkg)

    def call():
        with pytest.raises(M.B2SError) as e:
            O.OccupancyGrid(abi.laser_from(laser), ranges, poses, 0.05, bbox=[0, 0, 1e6, 1e6])
        assert e.value.status == abi.B2S_ERR_TOO_LARGE
    return call


def occgrid_create_and_ros_map(pkg):
    O = pkg.load("occgrid")
    laser, poses, ranges = _scans(pkg)

    def call():
        g = O.OccupancyGrid(pkg.abi.laser_from(laser), ranges, poses, 0.05)
        g.ros_map()
        g.close()
    return call


def gmapping_ros_map(pkg):
    laser = pkg.synth.Laser()
    ang = laser.min_angle + np.arange(laser.n_readings) * laser.angular_resolution
    m = pkg.load("gmapping").GMap(-25, -25, 25, 25, 0.1)
    m.compute_map(pkg.synth.make_match_case(60).ranges, ang, (0.0, 0.0))
    return m.ros_map


def hector_map_ros_map(pkg):
    return pkg.load("hector").HectorMap(256, 256, 0.05).ros_map


def _hector(pkg, **kw):
    H = pkg.load("hector")
    laser, poses, ranges = _scans(pkg)
    scans = [H.scan_to_data_container(r, laser, 0.05) for r in ranges]
    return H.HectorSlam(resolution=0.05, size_x=512, size_y=512, levels=3, **kw), poses.astype(np.float32), scans


def hector_process_stream(pkg):
    g, poses, scans = _hector(pkg)
    return lambda: g.process_stream(scans, (0, 0), first_hint=poses[0])


def hector_update_batch(pkg):
    g, poses, scans = _hector(pkg, batch=2)
    return lambda: g.update_batch(scans[:2], (0, 0), poses[:2])


def plicp_match(pkg):
    laser = pkg.synth.Laser()
    case = pkg.synth.make_match_case(7)
    theta = laser.min_angle + np.arange(laser.n_readings) * laser.angular_resolution
    return lambda: pkg.load("plicp").match(pkg.abi.icp_params(), [case.base_ranges], [case.ranges], theta, 0.1, 30.0,
                                           [[0, 0, 0]])


def deskew_undistort(pkg):
    DS = pkg.load("deskew")
    case = dc.make_case(pkg, 3)
    info = case["info"]
    info.imu_last, t, x, y, z = DS.integrate_imu(case["imu_stamps"], case["imu_ang"], info.time_start, case["t_end"])
    info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = DS.odom_increment(case["start_pose"], case["end_pose"])
    info.use_imu = info.use_odom = 1
    return lambda: DS.undistort(case["ranges"][None, :], case["angle_min"], case["angle_increment"], [info],
                                t[None], x[None], y[None], z[None])


def add_scans_degenerate_smear(pkg):
    """smear deviation = 10 x resolution: the smear kernel is 100 next to its centre, AddScan is order-dependent and runs
    the sequential kernel with its stream-ordered scratch"""
    M, abi, synth = pkg.load("matcher"), pkg.abi, pkg.synth
    cases = [synth.make_match_case(s) for s in (900, 901)]
    m = M.ScanMatcher(abi.matcher_params(1.5, 0.05, 0.5, 9.25), abi.laser_from(synth.Laser()), max_batch=2)
    m.set_scans(np.stack([c.ranges for c in cases]), np.stack([c.odom_pose for c in cases]))
    bran = np.stack([c.base_ranges for c in cases])[:, None, :]
    bpos = np.stack([c.base_pose for c in cases])[:, None, :]
    return lambda: m.add_scans(bran, bpos)


CASES = [occgrid_too_large, occgrid_create_and_ros_map, gmapping_ros_map, hector_map_ros_map, hector_process_stream,
         hector_update_batch, plicp_match, deskew_undistort, add_scans_degenerate_smear]


@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__)
def test_call_returns_its_pool_memory(pkg, case):
    assert pkg.load("matcher").device_count() > 0
    call = case(pkg)
    call()  # first call: module loading, pool set-up
    pool = _DefaultPool()
    before = pool.used()
    call()
    assert pool.used() == before
