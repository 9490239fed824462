"""Shared synthetic inputs of the lesson5 de-skew tests: a 10 Hz scan of n beams during which the sensor turns and
drives, 200 Hz IMU messages and two odometry messages bracketing the scan."""
import numpy as np


def make_case(pkg, seed, n=1081, rate=(0.6, -0.2, 0.9), vel=(0.8, 0.1, 0.0), dropouts=True):
    DS = pkg.load("deskew")
    rng = np.random.default_rng(seed)
    t0 = 100.0 + rng.uniform(0, 5)
    dt = 0.1 / n
    ranges = rng.uniform(0.5, 25.0, n).astype(np.float32)
    if dropouts:
        ranges[rng.integers(0, n, 20)] = np.inf
        ranges[rng.integers(0, n, 10)] = np.nan
        ranges[rng.integers(0, n, 10)] = 0.01
        ranges[:3] = np.inf  # the first VALID reading is not beam 0
    imu_t = t0 - 0.05 + np.arange(45) * 0.005 + rng.uniform(0, 0.001)
    ang = np.asarray(rate)[None, :] * (1 + 0.1 * rng.standard_normal((45, 3)))
    t_end = t0 + dt * (n - 1)
    o_start, o_end = t0 - 0.013, t_end - 0.004
    start_pose = np.array([1.0, 2.0, 0.0, 0.0, 0.0, 0.3])
    d = o_end - o_start
    end_pose = start_pose + np.array([vel[0] * d, vel[1] * d, vel[2] * d, 0.0, 0.0, rate[2] * d])
    info = DS.DeskewScan()
    info.time_start, info.time_increment = t0, dt
    info.range_min, info.range_max = 0.1, 30.0
    info.use_imu = info.use_odom = 1
    info.odom_start_time, info.odom_end_time = o_start, o_end
    return dict(ranges=ranges, angle_min=-2.35619449, angle_increment=4.71238898 / (n - 1), info=info, imu_stamps=imu_t,
                imu_ang=ang, t_end=t_end, start_pose=start_pose, end_pose=end_pose)


# ---------------------------------------------------------------- message streams for the unmodified node (ref_lesson5)

T0_SEC, T0_NSEC = 1000, 123456789


def to_sec(sec, nsec):
    """ros::Time::toSec"""
    return float(sec) + 1e-9 * float(nsec)


def _stamp(t_ns):
    return int(t_ns // 10 ** 9), int(t_ns % 10 ** 9)


def _quat(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = (np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(yaw / 2),
                              np.sin(yaw / 2))
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


def stream(n, n_scans, seed, angle_min=-2.35619449, angle_increment=None, time_increment=None, range_min=0.1,
           range_max=30.0, first_valid=(), imu_period_ns=5_000_000, imu_gap=None, odom_from_ns=-200_000_000,
           imu_at=None, rate=(7.0, -6.0, 25.0), special=None):
    """A recording at 10 Hz: n_scans LaserScans of n beams, IMU messages every imu_period_ns (or at the offsets imu_at
    returns for each scan), odometry at 50 Hz with 3-D motion.  Messages arrive at their stamps, a scan at the end of its
    sweep.  Times are integer nanoseconds from T0 so that every stamp is exact."""
    rng = np.random.default_rng(seed)
    ainc = np.float32(angle_increment if angle_increment is not None else (4.71238898 / (n - 1) if n > 1 else 0.0043633))
    tinc = np.float32(time_increment if time_increment is not None else 0.1 / max(n, 1))
    t0 = T0_SEC * 10 ** 9 + T0_NSEC
    period = 100_000_000
    dur_ns = int(np.ceil(float(tinc) * (n - 1) * 1e9)) + 1000
    ev, scans, starts = [], [], []
    for k in range(n_scans):
        s = t0 + k * period + int(rng.integers(0, 1000))
        starts.append(s)
        r = rng.uniform(0.5, 25.0, n).astype(np.float32)
        if n > 8:
            r[rng.integers(0, n, max(1, n // 50))] = np.inf
            r[rng.integers(0, n, max(1, n // 100))] = np.nan
        if k < len(first_valid):
            r[:first_valid[k]] = np.inf
        if special is not None:
            r = special(k, r)
        rmin, rmax = (range_min(k), range_max) if callable(range_min) else (range_min, range_max)
        fields = np.array([np.float32(angle_min), ainc, tinc, rmin, rmax], np.float32)
        scans.append((*_stamp(s), fields, r))
        ev.append((s + max(dur_ns, 0) + 1, ("scan", *_stamp(s), fields, r)))
    end = t0 + n_scans * period + 200_000_000
    if imu_at is None:
        stamps = range(t0 - 200_000_000 + 1_300_000, end, imu_period_ns)
    else:
        stamps = sorted(s + off for s in starts for off in imu_at)
    for ts in stamps:
        if imu_gap and imu_gap[0] <= ts - t0 < imu_gap[1]:
            continue
        x = (ts - t0) * 1e-9
        w = (rate[0] * np.cos(3 * x), rate[1] * (1 + 0.5 * np.sin(5 * x)), rate[2] * (1 + 0.2 * np.cos(2 * x)))
        ev.append((ts, ("imu", *_stamp(ts), w)))
    for ts in range(t0 + odom_from_ns + 700_000, end, 20_000_000):
        x = (ts - t0) * 1e-9
        pos = (3.0 + 1.5 * x, -2.0 - 0.7 * x, 0.1 + 0.3 * x)
        ev.append((ts, ("odom", *_stamp(ts), pos, _quat(0.3 * np.sin(2 * x), -0.2 * np.cos(3 * x), 2.5 + 0.8 * x))))
    ev.sort(key=lambda e: e[0])
    return dict(n=n, scans=scans, events=[e[1] for e in ev],
                imu=[(to_sec(*e[1][1:3]), e[1][3]) for e in ev if e[1][0] == "imu"],
                odom=[to_sec(*e[1][1:3]) for e in ev if e[1][0] == "odom"])


def _validity(k, r):
    """scan 0: [0.25, 20] with the edges and every non-finite; 1: range_min 0 with +-0 and a subnormal; 2: nothing valid"""
    lo, hi = np.float32(0.25), np.float32(20.0)
    sub = np.frombuffer(np.uint32(1).tobytes(), np.float32)[0]
    if k == 0:
        r[:12] = [lo, hi, np.nextafter(lo, np.float32(-1)), np.nextafter(hi, np.float32(np.inf)), -1.0, np.nan, np.inf,
                  -np.inf, sub, 0.0, -0.0, hi]
    elif k == 1:
        r[:8] = [0.0, -0.0, sub, -sub, np.nextafter(np.float32(0), np.float32(-1)), 5.0, np.nan, 20.0]
    elif k == 2:
        r[:] = np.where(np.arange(len(r)) % 2 == 0, np.inf, -1.0)
    return r


NODE_STREAMS = {
    # first valid beam at 0, 255, 256, 700 and n - 1 of a 1081-beam scan; roll and pitch to about 1.4 rad, yaw past pi
    "slabs": (dict(n=1081, n_scans=6, seed=1, first_valid=(0, 255, 256, 700, 1080)), (1, 1)),
    # a 1-beam scan has no duration, so no odometry message can fall inside it: IMU only
    **{f"beams{n}": (dict(n=n, n_scans=3, seed=10 + n, first_valid=(n - 1, 0)), (1, int(n > 1)))
       for n in (1, 2, 255, 256, 257, 4097)},
    "validity": (dict(n=24, n_scans=4, seed=3, range_min=lambda k: 0.0 if k == 1 else 0.25, range_max=20.0,
                      special=_validity), (1, 1)),
    **{f"flags{i}{o}": (dict(n=300, n_scans=3, seed=4), (i, o)) for i in (0, 1) for o in (0, 1)},
    # one IMU message 40 ms before each 40 ms scan and one 20 ms after it: imu_last = 0
    "imu_last0": (dict(n=100, n_scans=4, seed=5, time_increment=0.0004, imu_at=(-30_000_000, 60_000_000)), (1, 1)),
    "time_increment0": (dict(n=64, n_scans=3, seed=6, time_increment=0.0), (1, 0)),
    "angle_near_pi_negative_increment": (dict(n=720, n_scans=3, seed=7, angle_min=3.14159, angle_increment=-2 * np.pi / 720),
                                         (1, 1)),
    "angle_near_minus_pi": (dict(n=720, n_scans=3, seed=8, angle_min=-3.1415925, angle_increment=2 * np.pi / 720), (1, 1)),
    # odometry starts after scan 0 (dropped), IMU pauses across the end of scan 2 (dropped)
    "drops": (dict(n=200, n_scans=5, seed=9, odom_from_ns=50_000_000, imu_gap=(250_000_000, 420_000_000)), (1, 1)),
}
NODE_PUBLISHED = {"drops": [1, 3], "validity": [0, 1, 2], "slabs": [0, 1, 2, 3, 4], "imu_last0": [0, 1, 2]}


def node_answers(live):
    """{stream name: (stream, [published clouds])} from the unmodified node, live where oracle/_ref/ is built and replayed
    from tests/golden/reference/ elsewhere (one recording shared by the CPU and the GPU tests)."""
    from oracle import ref_lesson5
    from reference_record import Recording
    rec = Recording("test_deskew_reference__node_streams", live)
    out = {}
    for name, (kw, (use_imu, use_odom)) in NODE_STREAMS.items():
        st = stream(**kw)
        out[name] = (st, rec.value(name, lambda: ref_lesson5.run(st["events"], use_imu, use_odom),
                                   inputs=(st["events"], use_imu, use_odom)), (use_imu, use_odom))
    rec.save()
    return out


def abi_inputs(pkg, st, pub, flags):
    """The ABI inputs of one cloud the node published, built from the stream with the library's host preparation, and
    checked against the state the node computed that cloud from -> (scan index, ranges, angle_min, angle_increment,
    DeskewScan, (imu_time, rot_x, rot_y, rot_z))."""
    DS = pkg.load("deskew")
    k = [i for i, s in enumerate(st["scans"]) if (s[0], s[1]) == tuple(int(x) for x in pub["stamp"])][0]
    sec, nsec, fields, ranges = st["scans"][k]
    n = len(ranges)
    info = DS.DeskewScan()
    info.time_start, info.time_increment = to_sec(sec, nsec), float(fields[2])
    info.range_min, info.range_max = fields[3], fields[4]
    info.use_imu, info.use_odom = flags
    t_end = info.time_start + info.time_increment * (n - 1)
    assert pub["times"][0] == info.time_start and pub["times"][1] == t_end
    tab = [np.zeros(1)] * 4
    if flags[0]:
        msgs = [(t, w) for t, w in st["imu"] if not t < info.time_start - 0.1]  # PruneImuDeque's pruning
        last, *tab = DS.integrate_imu([m[0] for m in msgs], [m[1] for m in msgs], info.time_start, t_end)
        assert last == pub["imu_last"], (last, pub["imu_last"])
        for a, b in zip(tab, pub["imu"]):
            assert np.array_equal(a[:last + 1], b), "the library's IMU integration differs from the node's table"
        info.imu_last = last
        tab = [a[:last + 1] for a in tab]
    if flags[1]:
        before = [t for t in st["odom"] if t < info.time_start]
        inside = [t for t in st["odom"] if info.time_start <= t <= t_end]
        assert pub["times"][2] == before[-1] and pub["times"][3] == inside[-1]
        inc = DS.odom_increment(pub["poses"][0], pub["poses"][1])
        assert np.array_equal(inc.view(np.int32), pub["incre"].view(np.int32)), (inc, pub["incre"])
        info.odom_start_time, info.odom_end_time = pub["times"][2], pub["times"][3]
        info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = inc
    return k, ranges, float(fields[0]), float(fields[1]), info, tab


# ---------------------------------------------------------------- inputs only the ABI can express

def _abi_scan(pkg, rng, n, t0, tinc, use_imu=1, use_odom=1, odom=(None, None), incre=(0.4, -0.3, 0.1), first_valid=3):
    info = pkg.load("deskew").DeskewScan()
    info.time_start, info.time_increment, info.range_min, info.range_max = t0, tinc, 0.1, 30.0
    info.use_imu, info.use_odom = use_imu, use_odom
    os_, oe = odom
    info.odom_start_time = t0 - 0.013 if os_ is None else os_
    info.odom_end_time = t0 + tinc * (n - 1) - 0.004 if oe is None else oe
    info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = incre
    r = rng.uniform(0.5, 25.0, n).astype(np.float32)
    r[:first_valid] = np.inf
    return r, info


def _table(info, times, rots, stride=None, sentinel=0.0):
    """an IMU table of len(times) entries padded to stride with a sentinel (a read past imu_last would change the output)"""
    stride = stride or len(times)
    tab = [np.full(stride, sentinel, np.float64) for _ in range(4)]
    tab[0][:len(times)] = times
    for a in range(3):
        tab[a + 1][:len(times)] = np.asarray(rots)[:, a]
    info.imu_last = len(times) - 1
    return tab


AMIN, N_ABI = float(np.float32(-2.35619449)), 257
AINC = float(np.float32(4.71238898 / (N_ABI - 1)))


def _rots(rng, m, big=False):
    lim = (1.5, 1.5, 4.0) if big else (0.3, 0.3, 1.0)
    return np.stack([rng.uniform(-l, l, m) for l in lim], -1)


def _before_first_stamp(pkg):
    """negative time_increment: the beams run backwards in time, the later ones before imu_time[0] (front == 0)"""
    rng = np.random.default_rng(21)
    r, info = _abi_scan(pkg, rng, N_ABI, 50.0, -1e-4, odom=(49.97, 50.02))
    return [(r, AMIN, AINC, info, _table(info, [49.99, 50.0, 50.01, 50.03], _rots(rng, 4)))]


def _after_last_stamp(pkg):
    """the table ends inside the scan: later beams hold the last entry; imu_last 0 holds entry 0 throughout"""
    rng = np.random.default_rng(22)
    out = []
    for times in ([59.99, 60.004, 60.011], [59.995]):
        r, info = _abi_scan(pkg, rng, N_ABI, 60.0, float(np.float32(1e-4)))
        out.append((r, AMIN, AINC, info, _table(info, times, _rots(rng, len(times)))))
    return out


def _on_stamps(pkg):
    """table stamps equal to beam times: equality moves `front` past the stamp"""
    rng = np.random.default_rng(23)
    tinc = float(np.float32(1e-4))
    r, info = _abi_scan(pkg, rng, N_ABI, 20.0, tinc, first_valid=0)
    times = [20.0 - 0.001] + [20.0 + i * tinc for i in (0, 37, 128, 255)]
    return [(r, AMIN, AINC, info, _table(info, times, _rots(rng, 5)))]


def _sentinels(pkg):
    """imu_stride well past imu_last + 1, with non-zero entries after imu_last"""
    rng = np.random.default_rng(24)
    r, info = _abi_scan(pkg, rng, N_ABI, 30.0, float(np.float32(1e-4)))
    return [(r, AMIN, AINC, info, _table(info, [29.99, 30.006, 30.013], _rots(rng, 3), stride=16, sentinel=-7.5))]


def _odometry_inside_the_scan(pkg):
    """the odometry interval lies inside the scan: ratios below 0 and above 1"""
    rng = np.random.default_rng(25)
    r, info = _abi_scan(pkg, rng, N_ABI, 40.0, float(np.float32(1e-4)), odom=(40.008, 40.016), incre=(0.5, -0.25, 0.08))
    return [(r, AMIN, AINC, info, _table(info, [39.99, 40.01, 40.03], _rots(rng, 3)))]


def _flags_and_large_motion(pkg):
    """all four use_imu / use_odom combinations, roll and pitch to 1.5 rad and yaw past pi"""
    rng = np.random.default_rng(26)
    out = []
    for ui in (0, 1):
        for uo in (0, 1):
            r, info = _abi_scan(pkg, rng, N_ABI, 70.0, float(np.float32(1e-4)), use_imu=ui, use_odom=uo)
            times = 69.995 + np.arange(7) * 0.004
            out.append((r, AMIN, AINC, info, _table(info, times, _rots(rng, 7, big=True))))
    return out


ABI_CASES = {"before_first_stamp": _before_first_stamp, "after_last_stamp": _after_last_stamp, "on_stamps": _on_stamps,
             "sentinels": _sentinels, "odometry_inside_the_scan": _odometry_inside_the_scan,
             "flags_and_large_motion": _flags_and_large_motion}
