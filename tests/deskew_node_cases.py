"""Recordings for lesson5's whole de-skew node (b2s_lidar_undistortion_node, oracle/deskew_node_oracle.c): logs of
LaserScan, IMU and odometry messages with the number of IMU and odometry messages delivered before each scan's
callback, the conversion of such a recording into the message stream oracle/ref_lesson5.run feeds the unmodified node,
and the named recordings the tests share."""
import importlib

import numpy as np

import deskew_cases as dc

DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")
QUEUE_LENGTH = 2000


def from_events(events):
    """An event list as ref_lesson5.run takes it (delivery order) -> recording dict: amin, ainc, scans (SCAN_DTYPE with
    arrival counts), ranges [S, n] float32, imu (IMU_DTYPE), odom (ODOM_DTYPE)."""
    imu, odom, scans, ranges, counts = [], [], [], [], []
    for e in events:
        if e[0] == "imu":
            imu.append(((e[1], e[2]), e[3]))
        elif e[0] == "odom":
            odom.append(((e[1], e[2]), e[3], e[4]))
        else:
            scans.append(((e[1], e[2]), np.asarray(e[3], np.float32)))
            ranges.append(np.asarray(e[4], np.float32))
            counts.append((len(imu), len(odom)))
    f = np.stack([s[1] for s in scans])
    c = np.asarray(counts, np.int32).reshape(-1, 2)
    return dict(amin=np.float32(f[0, 0]), ainc=np.float32(f[0, 1]),
                scans=DS.node_scans([s[0] for s in scans], f[:, 2], f[:, 3], f[:, 4], c[:, 0], c[:, 1]),
                ranges=np.stack(ranges),
                imu=DS.imu_log(np.array([m[0] for m in imu], np.uint32).reshape(-1, 2), np.array([m[1] for m in imu]).reshape(-1, 3)),
                odom=DS.odom_log(np.array([m[0] for m in odom], np.uint32).reshape(-1, 2),
                                 np.array([m[1] for m in odom]).reshape(-1, 3), np.array([m[2] for m in odom]).reshape(-1, 4)))


def to_events(rec, n_callbacks=None):
    """A recording -> the event list of its first n_callbacks scan callbacks (all by default): before each scan, the
    IMU and odometry messages delivered by then, each log in its own order."""
    ev, i, o = [], 0, 0
    sc = rec["scans"]
    for k in range(len(sc) if n_callbacks is None else n_callbacks):
        for m in rec["imu"][i:sc[k]["imu_arrived"]]:
            ev.append(("imu", int(m["sec"]), int(m["nsec"]), tuple(float(x) for x in m["angular_velocity"])))
        for m in rec["odom"][o:sc[k]["odom_arrived"]]:
            ev.append(("odom", int(m["sec"]), int(m["nsec"]), tuple(float(x) for x in m["position"]),
                       tuple(float(x) for x in m["orientation"])))
        i, o = int(sc[k]["imu_arrived"]), int(sc[k]["odom_arrived"])
        fields = np.array([rec["amin"], rec["ainc"], sc[k]["time_increment"], sc[k]["range_min"], sc[k]["range_max"]],
                          np.float32)
        ev.append(("scan", int(sc[k]["sec"]), int(sc[k]["nsec"]), fields, rec["ranges"][k]))
    return ev


def _st(t_ns):
    return int(t_ns // 10 ** 9), int(t_ns % 10 ** 9)


def make(n=100, n_scans=6, seed=0, tinc=0.0004, jitter=True, imu_period=5_000_000, imu_skip=None, imu_extra=(),
         imu_arrival=None, odom_period=20_000_000, odom_first=-200_000_000, odom_quat=None, odom_latency=0,
         range_min=0.1, range_max=30.0):
    """A 10 Hz recording of n-beam scans built from stamps in integer nanoseconds after T0, each message delivered at
    its stamp (plus odom_latency, or at imu_arrival(index, stamp) for IMU) and each scan at the end of its sweep.
    imu_skip(rel_ns) drops IMU stamps, imu_extra adds some; odom_quat(index, rel_ns) overrides orientations."""
    rng = np.random.default_rng(seed)
    tinc = np.float32(tinc)
    t0 = dc.T0_SEC * 10 ** 9 + dc.T0_NSEC
    amin, ainc = np.float32(-2.35619449), np.float32(4.71238898 / max(n - 1, 1))
    dur = max(int(np.ceil(float(tinc) * (n - 1) * 1e9)), 0) + 1000
    ev = []
    for k in range(n_scans):
        s = t0 + k * 100_000_000 + (int(rng.integers(0, 1000)) if jitter else 0)
        r = rng.uniform(0.5, 25.0, n).astype(np.float32)
        if n > 8:
            r[rng.integers(0, n, max(1, n // 50))] = np.inf
        fields = np.array([amin, ainc, tinc, range_min, range_max], np.float32)
        ev.append((s + dur + 1, 1, ("scan", *_st(s), fields, r)))
    end = t0 + n_scans * 100_000_000 + 200_000_000
    stamps = [ts for ts in range(t0 - 200_000_000 + 1_300_000, end, imu_period) if not (imu_skip and imu_skip(ts - t0))]
    stamps = sorted(stamps + [t0 + x for x in imu_extra])
    for i, ts in enumerate(stamps):
        x = (ts - t0) * 1e-9
        w = (7.0 * np.cos(3 * x), -6.0 * (1 + 0.5 * np.sin(5 * x)), 25.0 * (1 + 0.2 * np.cos(2 * x)))
        ev.append((imu_arrival(i, ts - t0) + t0 if imu_arrival else ts, 0, ("imu", *_st(ts), w)))
    for i, ts in enumerate(range(t0 + odom_first + 700_000, end, odom_period)):
        x = (ts - t0) * 1e-9
        q = odom_quat(i, ts - t0) if odom_quat else None
        q = dc._quat(0.3 * np.sin(2 * x), -0.2 * np.cos(3 * x), 2.5 + 0.8 * x) if q is None else q
        ev.append((ts + odom_latency, 0, ("odom", *_st(ts), (3.0 + 1.5 * x, -2.0 - 0.7 * x, 0.1 + 0.3 * x), q)))
    ev.sort(key=lambda e: (e[0], e[1]))
    return [e[2] for e in ev]


def _late_bursts(rec):
    """IMU held back and delivered in bursts at every third scan callback: the scans between wait and are dropped"""
    c = rec["scans"]["imu_arrived"]
    rec["scans"]["imu_arrived"] = c[np.arange(len(c)) // 3 * 3]
    return rec


def _pitch90(i, rel):
    """every third odometry message at pitch +-90 degrees, unnormalised so that m[2][0] is exactly -+1"""
    return [(1.0, 1.0, -1.0, 1.0), (1.0, -1.0, 1.0, 1.0), (0.0, 1.0, 0.0, 1.0), None, None, None][i % 6]


def _swap_arrivals(i, rel):
    """IMU 58 and 59 (inside scan 1's sweep) arrive swapped; IMU 84 (inside scan 2) arrives just before scan 3's
    callback, after later stamps: the back of the queue is then older than scan 2's end"""
    if i == 58:
        return rel + 5_000_001
    if i == 59:
        return rel - 5_000_001
    if i == 84:
        return 339_000_000
    return rel


STREAMS = {
    # name: (event list, (use_imu, use_odom), callbacks the node may be fed: None = all)
    **{f"node_{k}": (lambda kw=kw: dc.stream(**kw)["events"], flags, None) for k, (kw, flags) in dc.NODE_STREAMS.items()},
    "late_imu": (lambda: make(n_scans=10, seed=31), (1, 1), None),
    # no IMU message in [start - 0.1, start) of scan 2: the first message it integrates is after its start
    "imu_gap_start": (lambda: make(seed=32, imu_skip=lambda t: 80_000_000 <= t < 202_000_000), (1, 1), None),
    # no IMU message in [start - 0.1, end] of scan 2: imu_last -1
    "imu_gap_whole": (lambda: make(seed=33, imu_skip=lambda t: 95_000_000 <= t < 245_000_000), (1, 1), None),
    # 3 200 IMU messages inside scan 2's sweep: the node writes past its 2000-entry table, so it is fed only the
    # callbacks before the one that corrects scan 2
    "imu_over_2000": (lambda: make(n=64, seed=34, tinc=0.0005, jitter=False,
                                   imu_extra=tuple(range(200_000_001, 231_500_000, 10_000))), (1, 1), 3),
    "imu_out_of_order": (lambda: make(seed=35, imu_arrival=_swap_arrivals), (1, 1), None),
    # the first odometry message is stamped exactly at scan 0's start: start_odom_msg_ stays default (NaN cloud)
    "odom_at_first_start": (lambda: make(seed=36, jitter=False, odom_first=-700_000, odom_period=10_000_000), (1, 1), None),
    # odometry every 230 ms: scans without a message inside keep the previous end_odom_msg_
    "odom_sparse": (lambda: make(n_scans=10, seed=37, odom_period=230_000_000, odom_first=-300_000_000), (1, 1), None),
    "odom_pitch90": (lambda: make(seed=38, odom_quat=_pitch90, odom_period=10_000_000), (1, 1), None),
    # beams run backwards over 0.2475 s; odometry delivered 250 ms late is all older than start - 0.1: pruned empty
    "negative_time_increment": (lambda: make(seed=39, tinc=-0.0025, odom_latency=250_000_000), (1, 1), None),
    **{f"mixed_flags{i}{o}": (lambda: make(n_scans=8, seed=40, odom_period=70_000_000, imu_skip=lambda t: 395_000_000 <= t < 545_000_000), (i, o), None)
       for i in (0, 1) for o in (0, 1)},
    "one_scan": (lambda: make(n_scans=1, seed=41), (1, 1), None),
    "two_scans": (lambda: make(n_scans=2, seed=42), (1, 1), None),
}
TRANSFORMS = {"late_imu": _late_bursts}


def recording(name):
    """-> (recording dict, flags, node callbacks)"""
    make_events, flags, callbacks = STREAMS[name]
    rec = from_events(make_events())
    rec = TRANSFORMS.get(name, lambda r: r)(rec)
    return rec, flags, callbacks


def restated(rec, flags, tables=False):
    from oracle import deskew_node_port
    return deskew_node_port.node(*flags, rec["amin"], rec["ainc"], rec["scans"], rec["ranges"], rec["imu"], rec["odom"],
                                 tables=tables)


def node_answers(live):
    """{name: (recording, flags, callbacks fed, [published clouds])} from the unmodified node, live where oracle/_ref/
    is built and replayed from tests/golden/reference/ elsewhere."""
    from oracle import ref_lesson5
    from reference_record import Recording
    rec_file = Recording("test_deskew_node_reference__node_streams", live)
    out = {}
    for name in STREAMS:
        rec, flags, callbacks = recording(name)
        ev = to_events(rec, callbacks)
        out[name] = (rec, flags, callbacks, rec_file.value(name, lambda: ref_lesson5.run(ev, *flags), inputs=(ev, *flags)))
    rec_file.save()
    return out


def same(a, b):
    """bit equality, NaN equal to NaN at any payload"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    iv = {4: np.int32, 8: np.int64}[a.dtype.itemsize]
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a).view(iv), np.where(nb, 0, b).view(iv))


def synthetic(n_scans, n, imu_hz=200, odom_hz=50, seed=0, tinc=None):
    """A long 10 Hz recording built with array operations: n_scans scans of n beams, IMU at imu_hz and odometry at
    odom_hz, each message delivered at its stamp and each scan at the end of its sweep (as `make` builds them)."""
    rng = np.random.default_rng(seed)
    t0 = dc.T0_SEC * 10 ** 9 + dc.T0_NSEC
    tinc = np.float32(0.1 / n if tinc is None else tinc)
    starts = t0 + np.arange(n_scans, dtype=np.int64) * 100_000_000 + rng.integers(0, 1000, n_scans)
    arrive = starts + max(int(np.ceil(float(tinc) * (n - 1) * 1e9)), 0) + 1000 + 1
    end = t0 + n_scans * 100_000_000 + 200_000_000
    its = np.arange(t0 - 200_000_000 + 1_300_000, end, 10 ** 9 // imu_hz, dtype=np.int64)
    ots = np.arange(t0 - 200_000_000 + 700_000, end, 10 ** 9 // odom_hz, dtype=np.int64)
    x, y = (its - t0) * 1e-9, (ots - t0) * 1e-9
    w = np.stack([7.0 * np.cos(3 * x), -6.0 * (1 + 0.5 * np.sin(5 * x)), 25.0 * (1 + 0.2 * np.cos(2 * x))], -1)
    q = np.stack(dc._quat(0.3 * np.sin(2 * y), -0.2 * np.cos(3 * y), 2.5 + 0.8 * y), -1)
    pos = np.stack([3.0 + 1.5 * y, -2.0 - 0.7 * y, 0.1 + 0.3 * y], -1)
    ranges = rng.uniform(0.5, 25.0, (n_scans, n)).astype(np.float32)
    ranges[rng.random((n_scans, n)) < 0.02] = np.inf
    st = lambda t: np.stack([t // 10 ** 9, t % 10 ** 9], -1)  # noqa: E731
    return dict(amin=np.float32(-2.35619449), ainc=np.float32(4.71238898 / max(n - 1, 1)),
                scans=DS.node_scans(st(starts), tinc, 0.1, 30.0, np.searchsorted(its, arrive, "right"),
                                    np.searchsorted(ots, arrive, "right")),
                ranges=ranges, imu=DS.imu_log(st(its), w), odom=DS.odom_log(st(ots), pos, q))
