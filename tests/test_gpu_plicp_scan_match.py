"""lesson3's scan-to-scan PL-ICP node on the device (b2s_plicp_scan_match_*) against the C restatement, which is pinned
to the unmodified node (tests/test_plicp_scan_match_reference.py), and against the library's own pair matcher.

Tolerance of the continuous outputs: 1e-9, the rule of test_gpu_plicp_odometry.py.  The device runs the restatement's
matcher operation for operation; only its sin / cos / atan2 / asin may differ from glibc's, by a few ulps (at most 3
measured, test_gpu_device_math.py), and a
scan whose match the float64 reference (plicp_reference.iterate) flags as borderline may take another decision there.
The pairs are independent, so such a scan is exempt alone: the scans after it must agree again."""
import ctypes as C
import math

import numpy as np
import pytest

import plicp_reference as pr
import plicp_scan_match_cases as sc

pytestmark = pytest.mark.gpu
TOL = 1e-9
DISCRETE = ("valid", "iterations", "nvalid", "matched")
CONT = ("x", "error", "theta_deg")


def _theta(rec):
    n = rec["ranges"].shape[1]
    return (rec["angle_min"] + np.arange(n, dtype=np.float32) * rec["angle_increment"]).astype(np.float64)


def _readings(rec, k):
    """Scan k as LaserScanToLDP sees it: float64 readings, NaN where the scan's own range fields reject them."""
    r = rec["ranges"][k].astype(np.float64)
    lo, hi = rec["limits"][k].astype(np.float64)
    with np.errstate(invalid="ignore"):
        return np.where((r > lo) & (r < hi), r, np.nan)


def _handle(pkg, recs, params=None):
    P = pkg.load("plicp")
    return P.ScanMatch(params if params is not None else sc.icp_params(recs[0]), [r["ranges"].shape[1] for r in recs],
                       [r["angle_min"] for r in recs], [r["angle_increment"] for r in recs])


def _alone(pkg, rec, params=None):
    h = _handle(pkg, [rec], params)
    out = h.process([rec["ranges"]], [rec["limits"]])[0]
    h.close()
    return out


def compare(rec, got, want, name):
    """Discrete outputs equal and continuous ones within TOL on every scan the float64 reference does not flag as
    borderline.  -> the exempted scans."""
    exempt = []
    P = sc.icp_params(rec)
    for k in range(len(want)):
        disc = all(got[k][f] == want[k][f] for f in DISCRETE)
        cont = all((np.isclose(np.asarray(got[k][f], np.float64), np.asarray(want[k][f], np.float64), rtol=0, atol=TOL,
                               equal_nan=True) | (got[k][f] == want[k][f])).all() for f in CONT)
        if disc and cont:
            continue
        assert k > 0, f"{name}: the initialising scan differs"
        _, _, _, _, flags = pr.iterate(P, _readings(rec, k - 1), _readings(rec, k), _theta(rec), -np.inf, np.inf,
                                       np.zeros(3), 1e-9)
        assert flags, f"{name} scan {k}: {[(f, got[k][f], want[k][f]) for f in DISCRETE + CONT]} with no borderline decision"
        exempt.append(k)
    return exempt


@pytest.fixture(scope="module")
def alone(pkg):
    """Every recording alone on a B = 1 handle."""
    return {name: _alone(pkg, rec) for name, rec in sc.STREAMS.items()}


@pytest.mark.parametrize("name", sorted(sc.STREAMS))
def test_device_equals_restatement(alone, name):
    """Every scan agrees except the ones the float64 reference flags as borderline; only recordings of identical
    or noise-free scans (exactly tied nearest neighbours) are expected to have any."""
    rec = sc.STREAMS[name]
    exempt = compare(rec, alone[name], sc.restate(rec), name)
    assert not exempt or name in ("identical", "odom_stop_and_go"), f"{name}: borderline scans {exempt}"


@pytest.mark.parametrize("name", sorted(n for n, r in sc.STREAMS.items() if len(r["ranges"]) > 1))
def test_each_scan_is_the_pair_matcher(pkg, alone, name):
    """b2s_plicp_match on (k - 1, k) from a zero guess returns scan k's result bit for bit: the node runs the pair
    kernel's matcher."""
    P = pkg.load("plicp")
    rec, got = sc.STREAMS[name], alone[name]
    S = len(got)
    ref = np.stack([_readings(rec, k - 1) for k in range(1, S)])
    cur = np.stack([_readings(rec, k) for k in range(1, S)])
    x, valid, it, nv, err = P.match(sc.icp_params(rec), ref, cur, _theta(rec), -np.inf, np.inf, np.zeros((S - 1, 3)))
    g = got[1:]
    assert np.array_equal(x.view(np.int64), g["x"].view(np.int64))
    assert np.array_equal(err.view(np.int64), g["error"].view(np.int64))
    assert (valid == g["valid"]).all() and (it == g["iterations"]).all() and (nv == g["nvalid"]).all()
    deg = x[:, 2] * 180 / math.pi
    assert np.array_equal(deg.view(np.int64), g["theta_deg"].view(np.int64))


def _lasers():
    """Recordings of different lasers (beam counts and angle fields) at the node's default parameters."""
    d = math.radians
    wide = (np.float32(-math.pi / 2), np.float32(d(1.0 / 3.0)))
    narrow = (np.float32(d(-60.0)), np.float32(d(0.6)))
    out = {n: sc.STREAMS[n] for n in ("odom_straight", "odom_backward", "odom_stop_and_go", "edges", "limits_change",
                                       "full_circle", "two_scans", "one_scan")}
    out["wide_541"] = sc.recording(sc.drive(41, [(0.02, 0.0, d(0.8))] * 9, n=541, laser=wide), laser=wide)
    out["narrow_200"] = sc.recording(sc.drive(42, [(0.02, 0.01, d(-0.5))] * 12, n=200, laser=narrow), laser=narrow)
    return out


def _same(a, b):
    return a.tobytes() == b.tobytes()


def test_chunking_and_reset(pkg):
    """One call, halves, uneven chunks and one scan per call (other recordings idle in some calls) give the same bytes;
    reset() restarts one recording, or all, as on a fresh handle."""
    pool = _lasers()
    names = sorted(pool)
    recs = [pool[n] for n in names]
    B = len(recs)
    h = _handle(pkg, recs, pkg.abi.icp_params())
    whole = h.process([r["ranges"] for r in recs], [r["limits"] for r in recs])

    def run(cuts):  # cuts[b] = increasing split points of recording b, the same number of calls for all
        h.reset()
        parts = [[] for _ in range(B)]
        for c in range(len(cuts[0]) - 1):
            res = h.process([r["ranges"][cuts[b][c]:cuts[b][c + 1]] for b, r in enumerate(recs)],
                            [r["limits"][cuts[b][c]:cuts[b][c + 1]] for b, r in enumerate(recs)])
            for b in range(B):
                parts[b].append(res[b])
        return [np.concatenate(p) for p in parts]

    L = [len(r["ranges"]) for r in recs]
    rng = np.random.default_rng(5)
    for cuts in ([[0, l // 2, l] for l in L],
                 [[0, min(3, l), min(3, l) + (b % 4), l] for b, l in enumerate(L)],
                 [[0] + [min(k, l) for k in range(1, max(L) + 1)] for l in L],
                 [[0] + [min(max(0, k - b), l) for k in range(1, max(L) + B + 1)] for b, l in enumerate(L)],
                 [[0] + sorted(rng.integers(0, l + 1, 5).tolist()) + [l] for l in L]):
        got = run(cuts)
        for b in range(B):
            assert _same(got[b], whole[b]), (names[b], cuts[b])
    h.reset()
    first = h.process([r["ranges"][:3] for r in recs], [r["limits"][:3] for r in recs])
    h.reset(2)
    rest = h.process([r["ranges"][3:] if b != 2 else r["ranges"] for b, r in enumerate(recs)],
                     [r["limits"][3:] if b != 2 else r["limits"] for b, r in enumerate(recs)])
    for b in range(B):
        got = rest[b] if b == 2 else np.concatenate([first[b], rest[b]])
        assert _same(got, whole[b]), names[b]
    h.close()


@pytest.mark.parametrize("B", [1, 7, 132])
def test_fleet_independence(pkg, B):
    """B ragged recordings of different lasers in one call: each equals the same recording alone on a B = 1 handle."""
    pool = _lasers()
    names = sorted(pool)
    P = pkg.abi.icp_params()
    ref = {n: _alone(pkg, pool[n], P) for n in names}
    recs = []
    for b in range(B):
        n = names[(b * 3) % len(names)]
        L = len(pool[n]["ranges"])
        recs.append((n, (b * 7 + 3) % (L + 1)))  # prefixes of 0 .. L scans
    h = _handle(pkg, [pool[n] for n, _ in recs], P)
    got = h.process([pool[n]["ranges"][:l] for n, l in recs], [pool[n]["limits"][:l] for n, l in recs])
    h.close()
    for b, (n, l) in enumerate(recs):
        assert _same(got[b], ref[n][:l]), (b, n, l)


@pytest.mark.parametrize("n", [3, 4, 1081, 2408])
def test_beam_counts(pkg, n):
    """The handle runs at 3, 4, 1081 and 2408 beams (the pair kernel's limit on an H100) and equals the restatement."""
    base = sc.STREAMS["odom_straight"]
    r = base["ranges"][:10]
    rec = sc.recording(np.ascontiguousarray(np.resize(r, (len(r), n)) if n != 1081 else r))
    compare(rec, _alone(pkg, rec), sc.restate(rec), f"n={n}")


def test_too_many_beams_refused(pkg):
    M = pkg.load("matcher")
    amin, ainc = sc.HOKUYO
    with pytest.raises(M.B2SError) as e:
        pkg.load("plicp").ScanMatch(pkg.abi.icp_params(), [1081, 2409, 5], [amin] * 3, [ainc] * 3)
    assert e.value.status == pkg.abi.B2S_ERR_TOO_LARGE


def test_invalid_arguments_write_nothing(pkg):
    """Refused calls return BAD_PARAMS, leave the output untouched and do not change the handle's state."""
    P = pkg.load("plicp")
    abi = pkg.abi
    L = P._bind()
    pool = _lasers()
    recs = [pool["odom_straight"], pool["wide_541"]]
    h = _handle(pkg, recs, abi.icp_params())
    first = h.process([recs[0]["ranges"][:4], recs[1]["ranges"][:4]], [recs[0]["limits"][:4], recs[1]["limits"][:4]])
    rng = np.ascontiguousarray(np.concatenate([recs[0]["ranges"][4:6].ravel(), recs[1]["ranges"][4:6].ravel()]))
    lim = np.ascontiguousarray(np.concatenate([recs[0]["limits"][4:6], recs[1]["limits"][4:6]]))
    out = (abi.PlicpScanMatchStep * 4)()
    C.memset(out, 0x5A, C.sizeof(out))
    sentinel = bytes(out)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    good = np.array([2, 2], np.int32)
    for counts, r, l in ((np.array([2, -1], np.int32), rng, lim), (good, None, lim), (good, rng, None)):
        rc = L.b2s_plicp_scan_match_process(h._h, counts.ctypes.data_as(ip),
                                            None if r is None else r.ctypes.data_as(fp),
                                            None if l is None else l.ctypes.data_as(fp), out)
        assert rc == abi.B2S_ERR_BAD_PARAMS
        assert bytes(out) == sentinel
    assert L.b2s_plicp_scan_match_process(h._h, None, rng.ctypes.data_as(fp), lim.ctypes.data_as(fp), out) == \
        abi.B2S_ERR_BAD_PARAMS
    assert L.b2s_plicp_scan_match_process(h._h, good.ctypes.data_as(ip), rng.ctypes.data_as(fp),
                                          lim.ctypes.data_as(fp), None) == abi.B2S_ERR_BAD_PARAMS
    for bad in (-2, 2, 100):
        assert L.b2s_plicp_scan_match_reset(h._h, bad) == abi.B2S_ERR_BAD_PARAMS
    assert bytes(out) == sentinel
    # the state is as the first call left it: the next scans continue the recordings
    rest = h.process([recs[0]["ranges"][4:], recs[1]["ranges"][4:]], [recs[0]["limits"][4:], recs[1]["limits"][4:]])
    h.close()
    for b in range(2):
        assert _same(np.concatenate([first[b], rest[b]]), _alone(pkg, recs[b], abi.icp_params())), b
