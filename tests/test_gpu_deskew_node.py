"""lesson5's whole de-skew node on the device (b2s_lidar_undistortion_node) against the C restatement
(oracle/deskew_node_oracle.c, pinned to the unmodified node by tests/test_deskew_node_reference.py): statuses, states
and clouds bit for bit on every named recording, every published row against b2s_lidar_undistort, a recording of more
than 65 537 scans, and IMU tables near the node's 2000 entries, which need more than 48 KB of shared memory."""
import importlib

import numpy as np
import pytest

import deskew_node_cases as nc

pytestmark = pytest.mark.gpu
DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")


def _device(rec, flags):
    return DS.undistort_recording(*flags, rec["amin"], rec["ainc"], rec["scans"], rec["ranges"], rec["imu"], rec["odom"])


def _check_equal(rec, flags, name):
    status, state, xyz = _device(rec, flags)
    want = nc.restated(rec, flags)
    assert np.array_equal(status, want["status"]), (name, list(status), list(want["status"]))
    for f in DS.STATE_DTYPE.names:
        assert nc.same(state[f], want["state"][f]), f"{name}: the per-scan states' {f} differs"
    for j in range(len(status)):
        assert nc.same(xyz[j], want["xyz"][j]), f"{name}: scan {j} ({status[j]}) cloud differs from the restatement"
    return status, state, xyz


@pytest.mark.parametrize("name", list(nc.STREAMS))
def test_device_equals_restatement(pkg, name):
    """Statuses, states and clouds: NaN equal to NaN at any payload, everything else by bits."""
    assert pkg.load("matcher").device_count() > 0
    rec, flags, _ = nc.recording(name)
    _check_equal(rec, flags, name)


def _pruned_queues(rec, flags, status, state):
    """{row: (first, end) of the IMU log in the node's queue after PruneImuDeque}, from the statuses"""
    if not flags[0]:
        return {}
    t = rec["imu"]["sec"].astype(np.float64) + 1e-9 * rec["imu"]["nsec"].astype(np.float64)
    starts = rec["scans"]["sec"].astype(np.float64) + 1e-9 * rec["scans"]["nsec"].astype(np.float64)
    lo, out = 0, {}
    for j, s in enumerate(status):
        if s in (DS.HELD, DS.WAIT_IMU):
            continue
        hi, start = int(rec["scans"]["imu_arrived"][j + 1]), starts[j]
        while lo < hi and t[lo] < start - 0.1:
            lo += 1
        out[j] = (lo, hi)
    return out


@pytest.mark.parametrize("name", list(nc.STREAMS))
def test_published_rows_equal_the_batch_call(pkg, name):
    """Every published row equals b2s_lidar_undistort fed the row's state and b2s_deskew_integrate_imu's table over the
    pruned IMU queue (rows with imu_last -1 as imu_last 0 of that table, whose entry 0 is zero; rows whose odometry
    interval has zero length, which the batch call refuses, are skipped)."""
    rec, flags, _ = nc.recording(name)
    status, state, xyz = _device(rec, flags)
    n = rec["ranges"].shape[1]
    queues = _pruned_queues(rec, flags, status, state)
    rows, infos, tabs = [], [], []
    for j in np.flatnonzero(status == DS.PUBLISHED):
        st = state[j]
        if st["use_odom"] and st["odom_start_time"] == st["odom_end_time"]:
            continue
        info = DS.DeskewScan.from_buffer_copy(st.tobytes())
        tab = [np.zeros(1)] * 4
        if flags[0]:
            lo, hi = queues[j]
            t = rec["imu"]["sec"][lo:hi].astype(np.float64) + 1e-9 * rec["imu"]["nsec"][lo:hi].astype(np.float64)
            end = st["time_start"] + st["time_increment"] * (n - 1)
            last, *tab = DS.integrate_imu(t, rec["imu"]["angular_velocity"][lo:hi], st["time_start"], end)
            assert last == st["imu_last"], (name, j, last, st["imu_last"])
            info.imu_last = max(last, 0)
        rows.append(j)
        infos.append(info)
        tabs.append(tab)
    if not rows:
        return
    stride = max(len(t[0]) for t in tabs)
    T = [np.stack([np.pad(t[a], (0, stride - len(t[a]))) for t in tabs]) for a in range(4)]
    got = DS.undistort(rec["ranges"][rows], rec["amin"], rec["ainc"], infos, *T)
    for b, j in enumerate(rows):
        assert nc.same(got[b], xyz[j]), f"{name}: scan {j} differs from b2s_lidar_undistort"


def test_more_than_65537_scans(pkg):
    """65 600 scans of 4 beams with 200 Hz IMU and 50 Hz odometry: published scans sit on grid x past 65 535."""
    rec = nc.synthetic(65_600, 4, seed=5)
    status, _, _ = _check_equal(rec, (1, 1), "65600 scans")
    assert (status == DS.PUBLISHED).sum() > 65_537


def test_imu_tables_near_2000_entries(pkg):
    """1081-beam scans with 20 kHz IMU: about 2000 table entries per scan, 64 KB of shared memory per CTA."""
    rec = nc.synthetic(6, 1081, imu_hz=20_000, seed=6)
    status, state, _ = _check_equal(rec, (1, 1), "20 kHz IMU")
    pub = status == DS.PUBLISHED
    assert pub.sum() == 5 and state["imu_last"][pub].max() + 1 > 48 * 1024 // 32
