"""lesson1's corner picker (LaserScan::ScanCallback, feature_detection.cc:77-179).  PARITY PINNED: the C++ restatement
(oracle/feature_oracle.cpp) is compared bit for bit with the unmodified node compiled against a ROS stand-in
(oracle/ref_lesson1.cpp), live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere.  The restated
libstdc++ introsort (csrc/introsort.cuh) is checked against the host's std::sort.  No GPU here: argument checks and
the refusal to run without a device."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import feature_cases as fc
from oracle import features_port as fp, ref_lesson1 as rl
from reference_record import digest, recording

HERE = os.path.dirname(os.path.abspath(__file__))

FAMILIES = {
    "rooms": lambda: fc.rooms(11, 60),
    "millimetre": lambda: fc.quantised(12, 60, 0.001),
    "centimetre": lambda: fc.quantised(13, 60, 0.01),
    "tie_heavy": lambda: fc.tie_heavy(14, 300),
    "full_width": lambda: fc.full_width(15, 20),
    "signed": lambda: fc.signed(16, 60),
    "huge": lambda: fc.huge(17, 60),
    "killer": fc.killer_scans,
}


def node_equals_restatement(rec, x, rec_name="node"):
    """the restatement's published ranges against the node's, all 1500 of them; returns the restatement's result"""
    res = fp.detect(x)
    n = x.shape[1]
    assert (res.count >= 0).all()
    mine = np.zeros((len(x), fp.MAX_BEAMS), np.float32)
    mine[:, :n] = res.ranges
    def live():
        ref = rl.detect(x)
        bad = np.flatnonzero((ref.view(np.int32) != mine.view(np.int32)).any(axis=1))
        assert bad.size == 0, f"restatement differs from the node on scans {bad[:10]}"
        return digest(ref)
    want = rec.value(rec_name, live, inputs=x)
    assert want == digest(mine), "restatement differs from the node's recorded answer"
    return res


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_restatement_equals_node(request, family):
    x = FAMILIES[family]()
    with recording(request, rl.available()) as rec:
        res = node_equals_restatement(rec, x)
    tied = (res.tied != 0).sum()
    if family == "rooms":
        assert tied == 0 and res.count.min() > 0  # natural scans: the cut decides without the sort order
    if family in ("tie_heavy", "huge"):
        assert tied >= len(x) // 2, tied  # the picks depend on std::sort's order among equal values
    if family == "killer":
        assert (res.heap >= 1).all(), res.heap  # every killer sector's sort fell back to heap sort
        assert list(res.tied) == [1 << 2, 1 << 4, 0]  # two with a tied cut in the killed sector, one without


def test_restatement_equals_node_short_scans(request):
    """every count of finite readings 0 .. 40: sectors that are skipped (s >= e), one entry long, or all placeholders"""
    with recording(request, rl.available()) as rec:
        for count, x in fc.short_scans(18):
            res = node_equals_restatement(rec, x, rec_name=f"count{count}")
            if count < 11:
                assert (res.count == 0).all()


def test_killer_fixture_matches_its_recipe():
    """tests/golden/feature_killer.npz is solve_killer_scan's output up to rounding: the same order of curvature"""
    k = fc.killer_scans()
    for i, (sector, huge_at) in enumerate(fc.KILLER_SPECS):
        again = fc.solve_killer_scan(sector, huge_at, seed=i)
        c0, c1 = fp.detect(k[i]).curvature[0], fp.detect(again).curvature[0]
        s, e = 1500 * sector // 6, 1500 * (sector + 1) // 6 - 1
        assert np.array_equal(np.argsort(c0[s:e], kind="stable"), np.argsort(c1[s:e], kind="stable"))


def test_curvature_is_the_left_to_right_float_stencil():
    """c at the beam of v[i], 5 <= i < count - 5, summed left to right in float32; NaN at every other beam"""
    x = fc.rooms(19, 3)
    res = fp.detect(x)
    for b in range(len(x)):
        beams = np.flatnonzero(np.isfinite(x[b]))
        v = x[b, beams]
        want = np.full(x.shape[1], np.nan, np.float32)
        for i in range(5, len(v) - 5):
            d = v[i - 5]
            for t in (-4, -3, -2, -1):
                d = np.float32(d + v[i + t])
            d = np.float32(d - np.float32(v[i] * np.float32(10)))
            for t in (1, 2, 3, 4, 5):
                d = np.float32(d + v[i + t])
            want[beams[i]] = np.float32(d * d)
        assert np.array_equal(res.curvature[b].view(np.int32), want.view(np.int32))


def test_nan_curvature_is_reported():
    x = fc.nan_curvature(20, 4)
    res = fp.detect(x)
    assert (res.count == -1).all() and not res.ranges.any()
    assert np.isnan(res.curvature).any()


def test_introsort_restatement_equals_std_sort(tmp_path):
    exe = str(tmp_path / "introsort_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(HERE, "introsort_check.cpp"), "-o", exe])
    out = json.loads(subprocess.check_output([exe, "300"], text=True))
    assert out["cases"] > 5000 and out["mismatches"] == 0, out
    assert out["killer_fallbacks"] > 200, out  # the heap-sort fallback is exercised, and agrees


def _raw(pkg, batch, n, ranges, thr, out, cnt=None, curv=None):
    L = pkg.load("features")._bind()
    fpp = C.POINTER(C.c_float)
    p = (lambda a: None if a is None else a.ctypes.data_as(fpp))
    return L.b2s_feature_detect(batch, n, p(ranges), thr, p(out),
                                None if cnt is None else cnt.ctypes.data_as(C.POINTER(C.c_int32)), p(curv), 0, None)


def test_argument_errors(pkg):
    abi = pkg.abi
    r, o = np.ones((2, 30), np.float32), np.zeros((2, 30), np.float32)
    assert _raw(pkg, 2, 30, None, 1.0, o) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(pkg, 2, 30, r, 1.0, None) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(pkg, -1, 30, r, 1.0, o) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(pkg, 2, -1, r, 1.0, o) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(pkg, 2, 30, r, -0.5, o) == abi.B2S_ERR_BAD_PARAMS
    assert _raw(pkg, 2, 30, r, float("nan"), o) == abi.B2S_ERR_BAD_PARAMS
    big = np.ones((1, 1501), np.float32)
    assert _raw(pkg, 1, 1501, big, 1.0, np.zeros_like(big)) == abi.B2S_ERR_TOO_LARGE
    with pytest.raises(ValueError):
        fp.detect(big)


def test_no_device_is_an_error(pkg):
    F, M = pkg.load("features"), pkg.load("matcher")
    if M.device_count() > 0:
        pytest.skip("a CUDA device is present; tests/test_gpu_features.py covers the device")
    for x in (np.ones((2, 30), np.float32), np.zeros((0, 30), np.float32), np.zeros((3, 0), np.float32)):
        with pytest.raises(M.B2SError) as e:
            F.detect(x)
        assert e.value.status == pkg.abi.B2S_ERR_NO_DEVICE
