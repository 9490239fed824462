"""lesson5's de-skew nodes behind one handle (b2s_deskew_node_*), fed in parts, against the C restatement
(oracle/deskew_node_oracle.c) and the one-shot call (b2s_lidar_undistortion_node): every named recording alone and
all of them in one handle, cut into calls anywhere (message split points included, calls without scans too), a fleet
of long recordings, reset, state that crosses calls, more than 65 537 rows and more than 48 KB of shared memory in one
launch, and refused calls that leave every node as it was.  Every comparison is bit for bit, NaN equal to NaN.

Rows of the handle are callback-indexed: row 0 of a recording is CACHED, row k >= 1 is the one-shot call's row k - 1."""
import importlib

import numpy as np
import pytest

import deskew_node_cases as nc

pytestmark = pytest.mark.gpu
DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")
NAMES = list(nc.STREAMS)


def _expected(rows):
    """one-shot rows (status, state, xyz) of a whole recording -> the handle's callback-indexed rows"""
    status, state, xyz = rows
    return (np.concatenate([[DS.CACHED], status[:-1]]).astype(np.int32), np.concatenate([np.zeros(1, DS.STATE_DTYPE), state[:-1]]),
            np.concatenate([np.zeros((1,) + xyz.shape[1:], np.float32), xyz[:-1]]))


def _restated(rec, flags):
    w = nc.restated(rec, flags)
    return _expected((np.asarray(w["status"], np.int32), w["state"], w["xyz"]))


def _one_shot(rec, flags):
    return _expected(DS.undistort_recording(*flags, rec["amin"], rec["ainc"], rec["scans"], rec["ranges"], rec["imu"],
                                            rec["odom"]))


def _check(got, want, name):
    assert np.array_equal(got[0], want[0]), (name, list(got[0]), list(want[0]))
    for f in DS.STATE_DTYPE.names:
        assert nc.same(got[1][f], want[1][f]), f"{name}: the states' {f} differs"
    assert got[2].shape == want[2].shape, name
    for k in range(len(got[0])):
        assert nc.same(got[2][k], want[2][k]), f"{name}: row {k} ({got[0][k]}) cloud differs"


def _random_cuts(rec, rng, max_chunk=5):
    """seeded chunk sizes 0 .. max_chunk (0: a call with messages and no scan), message split points drawn anywhere
    between the arrival counts of the scans around each cut"""
    S, cuts, at = len(rec["scans"]), [], 0
    while True:
        at += int(rng.integers(0, max_chunk + 1))
        if at >= S:
            break
        cuts.append(at)
    splits = []
    for field, n in (("imu_arrived", len(rec["imu"])), ("odom_arrived", len(rec["odom"]))):
        a = rec["scans"][field]
        m = [int(rng.integers(int(a[c - 1]) if c else 0, (int(a[c]) if c < S else n) + 1)) for c in cuts]
        splits.append(np.maximum.accumulate(m).tolist() if m else [])
    return cuts, splits[0], splits[1]


def _plans(rec, seed):
    """(label, chunks) cuttings of one recording: whole, one scan per call, and seeded random chunks"""
    S = len(rec["scans"])
    out = [("whole", DS.split_recording(rec, [])), ("per_scan", DS.split_recording(rec, range(1, S)))]
    rng = np.random.default_rng(seed)
    for r in range(3):
        out.append((f"random{r}", DS.split_recording(rec, *_random_cuts(rec, rng))))
    return out


def _feed(h, plans, rng=None):
    """Feed every recording its chunks through h, advancing a random subset of recordings per call when rng is given
    (else all together); -> per recording the concatenated (status, state, xyz)."""
    B = len(plans)
    pos, got = [0] * B, [[] for _ in range(B)]
    while any(pos[b] < len(plans[b]) for b in range(B)):
        chunks = [None] * B
        for b in range(B):
            if pos[b] < len(plans[b]) and (rng is None or rng.random() < 0.6):
                chunks[b] = plans[b][pos[b]]
                pos[b] += 1
        for b, r in enumerate(h.process(chunks)):
            if chunks[b] is not None:
                got[b].append(r)
    return [tuple(np.concatenate([r[i] for r in g]) for i in range(3)) for g in got]


@pytest.mark.parametrize("name", NAMES)
def test_each_recording_in_parts(pkg, name):
    """Each named recording with its own flags, whole, one scan per call and in random chunks: rows 1.. equal the
    restatement's rows 0..; row 0 is CACHED with zero bytes."""
    rec, flags, _ = nc.recording(name)
    want = _restated(rec, flags)
    for label, chunks in _plans(rec, seed=NAMES.index(name)):
        h = DS.DeskewNodeBatch([DS.laser_of(rec, flags)])
        _check(_feed(h, [chunks])[0], want, f"{name} {label}")
        h.close()


def test_all_recordings_in_one_handle(pkg):
    """Every named recording in one handle (beam counts and flags differ), each cut at random and advanced unevenly:
    every recording's rows equal its own restatement."""
    recs = [nc.recording(n)[:2] for n in NAMES]
    rng = np.random.default_rng(7)
    plans = [DS.split_recording(r, *_random_cuts(r, rng)) for r, _ in recs]
    h = DS.DeskewNodeBatch([DS.laser_of(r, f) for r, f in recs])
    got = _feed(h, plans, rng)
    assert len({r["ranges"].shape[1] for r, _ in recs}) > 1 and len({f for _, f in recs}) == 4
    for b, (r, f) in enumerate(recs):
        _check(got[b], _restated(r, f), NAMES[b])


def test_fleet_against_one_shot_calls(pkg):
    """132 recordings of 200 scans (541, 1081 and 1440 beams in turn, 200 Hz IMU) in chunks of 50 scans: each equals
    its own b2s_lidar_undistortion_node call."""
    recs = [nc.synthetic(200, (541, 1081, 1440)[b % 3], seed=100 + b) for b in range(132)]
    h = DS.DeskewNodeBatch([DS.laser_of(r, (1, 1)) for r in recs])
    got = _feed(h, [DS.split_recording(r, [50, 100, 150]) for r in recs])
    for b, r in enumerate(recs):
        want = _one_shot(r, (1, 1))
        assert (want[0] == DS.PUBLISHED).sum() > 150
        _check(got[b], want, f"fleet {b}")


def test_reset(pkg):
    """reset(b) mid-stream: b's later rows equal a fresh handle's fed the same chunks, the others are untouched;
    reset(-1) makes every recording fresh."""
    names = ["late_imu", "odom_sparse", "mixed_flags10"]
    recs = [nc.recording(n)[:2] for n in names]
    lasers = [DS.laser_of(r, f) for r, f in recs]
    halves = [DS.split_recording(r, [len(r["scans"]) // 2]) for r, _ in recs]
    whole = [_restated(r, f) for r, f in recs]
    for target in (1, -1):
        h = DS.DeskewNodeBatch(lasers)
        first = h.process([c[0] for c in halves])
        h.reset(target)
        later = h.process([c[1] for c in halves])
        fresh = DS.DeskewNodeBatch(lasers).process([c[1] for c in halves])
        for b in range(len(recs)):
            k = len(first[b][0])
            if target in (b, -1):
                _check(later[b], fresh[b], f"{names[b]} after reset({target})")
                assert later[b][0][0] == DS.CACHED
            else:
                _check(first[b], tuple(w[:k] for w in whole[b]), f"{names[b]} before")
                _check(later[b], tuple(w[k:] for w in whole[b]), f"{names[b]} untouched by reset({target})")


def test_state_carried_across_calls(pkg):
    """IMU bursts that straddle calls, a kept end_odom_msg_ across calls, and a call boundary inside an IMU gap."""
    rec, flags, _ = nc.recording("late_imu")
    want = _restated(rec, flags)
    assert (want[0] == DS.WAIT_IMU).any()
    for cuts in ([1, 2, 4, 5, 7, 8], [2, 3, 5, 6, 8, 9], list(range(1, 10))):
        a = rec["scans"]["imu_arrived"]
        mid = [(int(a[c - 1]) + int(a[c])) // 2 for c in cuts]  # bursts split between two calls
        _check(_feed(DS.DeskewNodeBatch([DS.laser_of(rec, flags)]), [DS.split_recording(rec, cuts, mid)])[0], want,
               f"late_imu {cuts}")

    rec, flags, _ = nc.recording("odom_sparse")
    want = _restated(rec, flags)
    got = _feed(DS.DeskewNodeBatch([DS.laser_of(rec, flags)]), [DS.split_recording(rec, range(1, len(rec["scans"])))])[0]
    _check(got, want, "odom_sparse per scan")
    pub = got[1]["odom_end_time"][got[0] == DS.PUBLISHED]
    assert (pub[1:] == pub[:-1]).any(), "no end_odom_msg_ was kept from one call to the next"

    rec, flags, _ = nc.recording("imu_gap_whole")
    want = _restated(rec, flags)
    for cuts in ([2], [2, 3], [1, 2, 3]):
        _check(_feed(DS.DeskewNodeBatch([DS.laser_of(rec, flags)]), [DS.split_recording(rec, cuts)])[0], want,
               f"imu_gap_whole {cuts}")


def test_more_than_65537_rows_in_one_call(pkg):
    """Three recordings of 22 000 four-beam scans in one call: more than 65 537 published rows on grid x."""
    recs = [nc.synthetic(22_000, 4, seed=s) for s in (11, 12, 13)]
    h = DS.DeskewNodeBatch([DS.laser_of(r, (1, 1)) for r in recs])
    got = h.process([DS.split_recording(r, [])[0] for r in recs])
    assert sum(int((g[0] == DS.PUBLISHED).sum()) for g in got) > 65_537
    for b, r in enumerate(recs):
        _check(got[b], _one_shot(r, (1, 1)), f"65537 rows {b}")


def test_large_imu_tables_with_small_ones(pkg):
    """A 1081-beam recording with 20 kHz IMU (about 2000 table entries, 64 KB of shared memory) in one launch with
    small-table recordings."""
    recs = [nc.synthetic(6, 1081, imu_hz=20_000, seed=21), nc.synthetic(6, 64, seed=22), nc.synthetic(9, 300, seed=23)]
    h = DS.DeskewNodeBatch([DS.laser_of(r, (1, 1)) for r in recs])
    got = h.process([DS.split_recording(r, [])[0] for r in recs])
    assert got[0][1]["imu_last"].max() + 1 > 48 * 1024 // 32
    for b, r in enumerate(recs):
        _check(got[b], _one_shot(r, (1, 1)), f"large tables {b}")


def _raw_args(h, chunks):
    """the arrays of one b2s_deskew_node_process call, as DeskewNodeBatch.process builds them"""
    sc = [np.asarray(c[0], DS.SCAN_DTYPE) for c in chunks]
    args = dict(n_scans=np.array([len(s) for s in sc], np.int32), scans=np.concatenate(sc),
                ranges=np.concatenate([np.asarray(c[1], np.float32).reshape(-1) for c in chunks]),
                n_imu=np.array([len(c[2]) for c in chunks], np.int32), imu=np.concatenate([c[2] for c in chunks]),
                n_odom=np.array([len(c[3]) for c in chunks], np.int32), odom=np.concatenate([c[3] for c in chunks]))
    total = len(args["scans"])
    args.update(out_status=np.full(total, 0x5A5A5A5A, np.int32),
                out_state=np.frombuffer(b"\x5a" * (total * DS.STATE_DTYPE.itemsize), DS.STATE_DTYPE).copy(),
                out_xyz=np.full(len(args["ranges"]) * 3, 7.5, np.float32))
    return args


ORDER = ["n_scans", "scans", "ranges", "n_imu", "imu", "n_odom", "odom", "out_status", "out_state", "out_xyz"]


def _call(h, args, **null):
    return DS._bind().b2s_deskew_node_process(h._h, *(None if null.get(k) else args[k].ctypes.data for k in ORDER))


def test_refusals_write_nothing(pkg):
    """Every refused call answers BAD_PARAMS and writes nothing; the next valid call equals the same call on a handle
    that never saw the refused ones."""
    recs = [nc.recording(n)[:2] for n in ("late_imu", "mixed_flags11")]
    lasers = [DS.laser_of(r, f) for r, f in recs]
    parts = [DS.split_recording(r, [3, 6]) for r, _ in recs]
    h, clean = DS.DeskewNodeBatch(lasers), DS.DeskewNodeBatch(lasers)
    h.process([p[0] for p in parts])
    clean.process([p[0] for p in parts])
    BAD = 1

    def refused(args, **null):
        before = {k: args[k].copy() for k in ("out_status", "out_state", "out_xyz")}
        assert _call(h, args, **null) == BAD
        for k, v in before.items():
            assert v.tobytes() == args[k].tobytes(), f"a refused call wrote {k}"

    for k in ("n_scans", "n_imu", "n_odom", "scans", "ranges", "imu", "odom", "out_status", "out_xyz"):
        refused(_raw_args(h, [p[1] for p in parts]), **{k: True})
    for k in ("n_scans", "n_imu", "n_odom"):
        a = _raw_args(h, [p[1] for p in parts])
        a[k][1] = -1
        refused(a)
    a = _raw_args(h, [p[1] for p in parts])
    a["scans"]["imu_arrived"][1] = a["scans"]["imu_arrived"][0] - 1 if a["scans"]["imu_arrived"][0] > 0 else -1
    refused(a)  # decreasing (or negative) IMU arrivals
    a = _raw_args(h, [p[1] for p in parts])
    a["scans"]["odom_arrived"][-1] = a["n_odom"][1] + 1
    refused(a)  # more odometry than the recording's log of the call
    a = _raw_args(h, [p[1] for p in parts])
    a["n_imu"][:] = 0
    a["scans"]["imu_arrived"] = 0
    refused(a, imu=True)  # a NULL log whose flag is on, though no message comes
    for bad in (2, -2):
        with pytest.raises(pkg.load("matcher").B2SError):
            h.reset(bad)
    got, want = h.process([p[1] for p in parts]), clean.process([p[1] for p in parts])
    for b in range(2):
        _check(got[b], want[b], f"after refusals {b}")
    got, want = h.process([p[2] for p in parts]), clean.process([p[2] for p in parts])
    for b in range(2):
        _check(got[b], want[b], f"after refusals, next call {b}")
