"""lesson1's corner picker on the device (b2s_feature_detect) against the C++ restatement (oracle/feature_oracle.cpp,
itself pinned to the unmodified node by tests/test_features.py): bit patterns equal for the published ranges, the
curvature (NaN positions included) and the pick count, on every family of tests/feature_cases.py."""
import numpy as np
import pytest

import feature_cases as fc
from oracle import features_port as fp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F(pkg):
    F, M = pkg.load("features"), pkg.load("matcher")
    if M.device_count() < 1:
        pytest.fail("no CUDA device")
    return F


def assert_same(F, x, thr=1.0, **kw):
    got, cnt, curv = F.detect(x, thr, **kw)
    want = fp.detect(x, thr)
    bad = np.flatnonzero((got.view(np.int32) != want.ranges.view(np.int32)).any(axis=1))
    assert bad.size == 0, f"published ranges differ on scans {bad[:10]} (tied-cut sectors {want.tied[bad[:10]]})"
    assert np.array_equal(cnt, want.count), np.flatnonzero(cnt != want.count)[:10]
    assert np.array_equal(curv.view(np.int32), want.curvature.view(np.int32)), "curvature differs"
    return want


FAMILIES = {
    "rooms": lambda: fc.rooms(31, 200),
    "millimetre": lambda: fc.quantised(32, 200, 0.001),
    "centimetre": lambda: fc.quantised(33, 200, 0.01),
    "tie_heavy": lambda: fc.tie_heavy(34, 500),
    "full_width": lambda: fc.full_width(35, 50),
    "signed": lambda: fc.signed(36, 200),
    "huge": lambda: fc.huge(37, 200),
    "killer": fc.killer_scans,
}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_device_equals_restatement(F, family):
    want = assert_same(F, FAMILIES[family]())
    tied = (want.tied != 0).sum()
    if family == "rooms":
        assert tied == 0  # only the rank-counting selection ran
    if family in ("tie_heavy", "huge", "killer"):
        assert tied > 0  # the device's introsort ran
    if family == "killer":
        assert (want.heap >= 1).all() and want.tied[0] and want.tied[1]  # ... and fell back to heap sort


def test_short_scans(F):
    for count, x in fc.short_scans(38):
        assert_same(F, x)


@pytest.mark.parametrize("thr", [0.0, 1.0, 1e30])
def test_thresholds(F, thr):
    x = np.concatenate([fc.rooms(39, 50), fc.tie_heavy(40, 50), fc.huge(41, 50, n=1081)])
    want = assert_same(F, x, thr)
    if thr == 1e30:
        assert want.count.max() > 0  # only infinite curvatures pass
    if thr == 0.0:
        assert want.count.min() > 0


def test_nan_curvature_among_normal_scans(F):
    x = np.concatenate([fc.rooms(42, 5)[:, :360], fc.nan_curvature(43, 3), fc.tie_heavy(44, 5, n=360)])
    x = x[np.random.default_rng(0).permutation(len(x))]
    want = assert_same(F, x)
    assert (want.count == -1).sum() == 3


@pytest.mark.parametrize("batch", [1, 7, 10000])
def test_batches(F, batch):
    """a batch equals its scans run one at a time (sampled rows for the large batch)"""
    x = np.concatenate([fc.rooms(45, batch - batch // 2), fc.tie_heavy(46, batch // 2)])
    x = x[np.random.default_rng(1).permutation(len(x))]
    got, cnt, curv = F.detect(x)
    rows = range(batch) if batch < 100 else np.random.default_rng(2).choice(batch, 40, replace=False)
    for b in rows:
        g1, c1, k1 = F.detect(x[b])
        assert np.array_equal(got[b].view(np.int32), g1[0].view(np.int32)) and cnt[b] == c1[0]
        assert np.array_equal(curv[b].view(np.int32), k1[0].view(np.int32))
    if batch < 100:
        assert_same(F, x)
    else:
        want = fp.detect(x[:500])
        assert np.array_equal(got[:500].view(np.int32), want.ranges.view(np.int32))
        assert np.array_equal(cnt[:500], want.count)


def test_optional_outputs_and_empty_calls(F):
    x = fc.tie_heavy(47, 9)
    got, cnt, curv = F.detect(x, want_curvature=False)
    assert curv is None and np.array_equal(got.view(np.int32), fp.detect(x).ranges.view(np.int32))
    g, c, k = F.detect(np.zeros((0, 100), np.float32))
    assert g.shape == (0, 100)
    g, c, k = F.detect(np.zeros((4, 0), np.float32))
    assert g.shape == (4, 0) and (c == 0).all()


def test_caller_stream(F):
    import torch
    x = np.concatenate([fc.rooms(48, 20), fc.tie_heavy(49, 20)])
    s = torch.cuda.Stream()
    got, cnt, curv = F.detect(x, stream=s.cuda_stream)
    want = fp.detect(x)
    assert np.array_equal(got.view(np.int32), want.ranges.view(np.int32)) and np.array_equal(cnt, want.count)
