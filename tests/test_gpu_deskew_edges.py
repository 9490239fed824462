"""lesson5 motion de-skew on the device (b2s_lidar_undistort) against the unmodified node, the C restatement and the
float64 reference (tests/deskew_reference.py), at the edges where the kernel could go wrong: beam counts around the
256-beam slab, first valid beams in every slab position, range edges, IMU tables searched off both ends and onto their
stamps, sentinels past imu_last, odometry ratios outside [0, 1], all use_imu / use_odom combinations in one batch,
large roll and pitch, and batches of 1, 3 and 65 537 scans.  The node's clouds replay from tests/golden/reference/
where oracle/_ref/ is absent."""
from collections import defaultdict

import numpy as np
import pytest

import deskew_cases as dc
import deskew_reference as dr
from oracle import port, ref_lesson5

pytestmark = pytest.mark.gpu


def _undistort(pkg, group, sentinel=-7.5):
    """One device call for scans sharing a beam count and angles: IMU tables padded to a common stride with a
    non-zero sentinel."""
    DS = pkg.load("deskew")
    stride = max(len(tab[0]) for _, _, _, _, tab in group)
    T, X, Y, Z = (np.full((len(group), stride), sentinel) for _ in range(4))
    for b, (_, _, _, _, tab) in enumerate(group):
        for dst, src in zip((T, X, Y, Z), tab):
            dst[b, :len(src)] = src
    r = np.stack([g[0] for g in group])
    return DS.undistort(r, group[0][1], group[0][2], [g[3] for g in group], T, X, Y, Z)


def _equal(a, b):
    return np.array_equal(a.view(np.int32), b.view(np.int32))


def test_device_equals_node(pkg):
    """Every cloud the node published, one device call per scan geometry: the same bits as the node and the
    restatement, and within the float64 bound."""
    assert pkg.load("matcher").device_count() > 0
    groups = defaultdict(list)
    for name, (st, pubs, flags) in dc.node_answers(ref_lesson5.available()).items():
        for pub in pubs:
            _, ranges, amin, ainc, info, tab = dc.abi_inputs(pkg, st, pub, flags)
            groups[(len(ranges), amin, ainc)].append(((ranges, amin, ainc, info, tab), pub["xyz"], name))
    assert len(groups) >= 8
    for key, items in groups.items():
        got = _undistort(pkg, [it[0] for it in items])
        for b, ((ranges, amin, ainc, info, tab), node, name) in enumerate(items):
            diff = got[b].view(np.int32) != node.view(np.int32)
            assert not diff.any(), f"{name}: {diff.any(1).sum()} beams differ from the node, first {np.argwhere(diff)[0]}"
            assert _equal(got[b], port.deskew_scan(ranges, amin, ainc, info, *tab)), name
            dr.check(got[b], ranges, amin, ainc, info, *tab)


def test_device_on_inputs_only_the_abi_expresses(pkg):
    """Hand-made IMU tables (before the first stamp, after the last, on the stamps), sentinels past imu_last, odometry
    ratios below 0 and above 1, mixed flags and large motion, all in one call: the restatement's bits and within the
    float64 bound."""
    group = [c for make in dc.ABI_CASES.values() for c in make(pkg)]
    assert len({c[3].imu_last for c in group}) >= 4  # a different imu_last per scan in one batch
    got = _undistort(pkg, group)
    for b, (ranges, amin, ainc, info, tab) in enumerate(group):
        assert _equal(got[b], port.deskew_scan(ranges, amin, ainc, info, *tab)), b
        dr.check(got[b], ranges, amin, ainc, info, *tab)


@pytest.mark.parametrize("batch", [1, 3, 65537])
def test_device_batch_sizes(pkg, batch):
    """Scans of 8 beams, each with its own stamps, ranges and IMU table: a batch past the 65 535 limit of a grid's y
    dimension is corrected like a small one."""
    DS = pkg.load("deskew")
    rng = np.random.default_rng(batch)
    n, stride = 8, 4
    amin, ainc = float(np.float32(-0.5)), float(np.float32(0.125))
    ranges = rng.uniform(0.5, 20.0, (batch, n)).astype(np.float32)
    ranges[::5, 0] = np.nan
    T = 10.0 + np.arange(batch)[:, None] * 0.1 + np.array([-0.01, 0.0003, 0.0005, 0.0008])[None, :]
    X, Y, Z = (rng.uniform(-0.5, 0.5, (batch, stride)) for _ in range(3))
    infos = []
    for b in range(batch):
        info = DS.DeskewScan()
        info.time_start, info.time_increment, info.range_min, info.range_max = 10.0 + b * 0.1, 1e-4, 0.1, 30.0
        info.use_imu, info.use_odom, info.imu_last = 1, b % 2, 1 + b % 3
        info.odom_start_time, info.odom_end_time = info.time_start - 0.01, info.time_start + 0.0005
        info.odom_incre[0], info.odom_incre[1], info.odom_incre[2] = 0.05, -0.02, 0.01
        infos.append(info)
    got = DS.undistort(ranges, amin, ainc, infos, T, X, Y, Z)
    for b in range(batch):
        assert _equal(got[b], port.deskew_scan(ranges[b], amin, ainc, infos[b], T[b], X[b], Y[b], Z[b])), b
    for b in sorted({0, batch // 2, batch - 1} | set(range(0, batch, 997))):
        dr.check(got[b], ranges[b], amin, ainc, infos[b], T[b], X[b], Y[b], Z[b])
