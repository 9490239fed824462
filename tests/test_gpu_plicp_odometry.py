"""lesson3's PL-ICP odometry node on the device (b2s_plicp_odom_*) against the C restatement, which is pinned to the
unmodified node (tests/test_plicp_odometry_reference.py), and against the library's own pair matcher.

Tolerance of the continuous outputs: 1e-9.  The device's tf chain is the restatement's operation for operation without
FMA contraction; only its sin / cos / atan2 / asin may differ from glibc's, by a few ulps (test_gpu_device_math.py
measures ros_math.cuh's composed results on the device at most 3 ulps from the correctly rounded ones, glibc's at most
1: ~1e-15 relative), and every scan's pose is a product of at most a few dozen such transforms since the first scan,
each correction further solved by a matcher whose iterations contract such differences.  1e-9 leaves six orders of
magnitude above that and is still far below anything a key-frame threshold or a published pose could notice."""
import numpy as np
import pytest

import plicp_odometry_cases as pc
import plicp_reference as pr

pytestmark = pytest.mark.gpu
TOL = 1e-9
DISCRETE = ("valid", "iterations", "nvalid", "published", "keyframe", "reference_scan")
CONT = ("position", "orientation", "linear", "angular", "first_guess", "x", "error")


def _odom(pkg, st, batch=1, n=None):
    P = pkg.load("plicp")
    return P.Odometry(pc.odom_params(st), batch, n or st["ranges"].shape[1], *map(float, pc.FIELDS))


def _theta(n):
    f = pc.FIELDS
    return (f[0] + np.arange(n, dtype=np.float32) * f[1]).astype(np.float64)


def _borderline(st, ref_steps, k):
    """The float64 reference's margins for scan k's match (from the restatement's first guess)."""
    P = pc.odom_params(st)
    kf = ref_steps[k]["reference_scan"]
    _, _, _, _, fl = pr.iterate(P.icp, st["ranges"][kf].astype(np.float64), st["ranges"][k].astype(np.float64),
                                _theta(st["ranges"].shape[1]), float(pc.FIELDS[2]), float(pc.FIELDS[3]),
                                ref_steps[k]["first_guess"], 1e-9)
    return fl


def compare(st, got, want, name):
    """Discrete outputs equal and continuous ones within TOL on every scan up to the first one the float64 reference
    flags as borderline (where a last-place difference may flip a decision; the recording may differ after it)."""
    for k in range(len(want)):
        if any(got[k][f] != want[k][f] for f in DISCRETE):
            flags = _borderline(st, want, k)
            assert flags, f"{name} scan {k}: {[(f, got[k][f], want[k][f]) for f in DISCRETE]} with no borderline decision"
            return k
        for f in CONT:
            a, b = np.asarray(got[k][f], np.float64), np.asarray(want[k][f], np.float64)
            ok = np.isclose(a, b, rtol=0, atol=TOL, equal_nan=True) | (a == b)
            assert ok.all(), f"{name} scan {k} {f}: {a} vs {b}"
    return len(want)


@pytest.fixture(scope="module")
def alone(pkg):
    """Every stream alone on a B = 1 handle."""
    out = {}
    for name, st in pc.STREAMS.items():
        o = _odom(pkg, st)
        out[name] = o.process([st["ranges"]], [st["stamps"]])[0]
        o.close()
    return out


@pytest.mark.parametrize("name", sorted(pc.STREAMS))
def test_device_equals_restatement(alone, name):
    """Every scan agrees up to the first borderline match, if any.  Only the noise-free stop-and-go stream (identical
    scans, so exactly tied nearest neighbours) is expected to reach one; every other stream agrees on every scan."""
    st = pc.STREAMS[name]
    upto = compare(st, alone[name], pc.restate(st), name)
    assert upto == len(st["ranges"]) or name == "stop_and_go", f"{name}: borderline at scan {upto}"


@pytest.mark.parametrize("name", sorted(pc.STREAMS))
def test_each_scan_is_the_pair_matcher(pkg, alone, name):
    """b2s_plicp_match on each scan's key frame, its ranges and its reported first guess returns its reported sm_icp
    result bit for bit: the odometry path runs the pair kernel's matcher."""
    P = pkg.load("plicp")
    st, got = pc.STREAMS[name], alone[name]
    ks = [k for k in range(len(got)) if got[k]["published"]]
    r = st["ranges"].astype(np.float64)
    x, valid, it, nv, err = P.match(pc.odom_params(st).icp, r[[got[k]["reference_scan"] for k in ks]], r[ks],
                                    _theta(r.shape[1]), float(pc.FIELDS[2]), float(pc.FIELDS[3]),
                                    np.stack([got[k]["first_guess"] for k in ks]))
    g = got[ks]
    assert np.array_equal(x.view(np.int64), g["x"].view(np.int64))
    assert np.array_equal(err.view(np.int64), g["error"].view(np.int64))
    assert (valid == g["valid"]).all() and (it == g["iterations"]).all() and (nv == g["nvalid"]).all()


def _fleet_params_stream():
    return pc.STREAMS["straight"]  # one parameter set and one mount for a whole handle


def _same(a, b):
    return a.tobytes() == b.tobytes()


def test_chunking_and_reset(pkg):
    """One call, halves, uneven chunks and one scan per call (other recordings idle in some calls) give the same bits;
    reset() restarts a recording as on a fresh handle."""
    names = ["straight", "backward", "stop_and_go", "scan_count", "jitter_stamps", "equal_stamps", "no_valid_reading"]
    recs = [pc.STREAMS[n] for n in names]
    B = len(recs)
    o = _odom(pkg, _fleet_params_stream(), B)
    whole = o.process([s["ranges"] for s in recs], [s["stamps"] for s in recs])

    def run(cuts):  # cuts[b] = increasing split points of recording b, same number of calls for all
        o.reset()
        parts = [[] for _ in range(B)]
        for c in range(len(cuts[0]) - 1):
            res = o.process([s["ranges"][cuts[b][c]:cuts[b][c + 1]] for b, s in enumerate(recs)],
                            [s["stamps"][cuts[b][c]:cuts[b][c + 1]] for b, s in enumerate(recs)])
            for b in range(B):
                parts[b].append(res[b])
        return [np.concatenate(p) for p in parts]

    L = [len(s["ranges"]) for s in recs]
    for cuts in ([[0, l // 2, l] for l in L],
                 [[0, min(3, l), min(3, l) + (b % 4), l] for b, l in enumerate(L)],
                 [[0] + [min(k, l) for k in range(1, max(L) + 1)] for l in L],
                 [[0] + [min(max(0, k - b), l) for k in range(1, max(L) + B + 1)] for b, l in enumerate(L)]):
        got = run(cuts)
        for b in range(B):
            assert _same(got[b], whole[b]), (names[b], cuts[b])
    # reset one recording mid-stream: its rerun equals the first run, the others continue untouched
    o.reset()
    first = o.process([s["ranges"][:5] for s in recs], [s["stamps"][:5] for s in recs])
    o.reset(2)
    rest = o.process([s["ranges"][5:] if b != 2 else s["ranges"] for b, s in enumerate(recs)],
                     [s["stamps"][5:] if b != 2 else s["stamps"] for b, s in enumerate(recs)])
    for b in range(B):
        got = rest[b] if b == 2 else np.concatenate([first[b], rest[b]])
        assert _same(got, whole[b]), names[b]
    o.close()


@pytest.mark.parametrize("B", [1, 7, 133, 1000])
def test_fleet_independence(pkg, B):
    """B recordings of different lengths in one call: each equals the same recording alone on a B = 1 handle."""
    base = _fleet_params_stream()
    pool = ["straight", "backward", "stop_and_go", "scan_count", "jitter_stamps", "equal_stamps", "no_valid_reading"]
    one = _odom(pkg, base)
    ref = {}
    for nme in pool:
        one.reset()
        ref[nme] = one.process([pc.STREAMS[nme]["ranges"]], [pc.STREAMS[nme]["stamps"]])[0]
    one.close()
    recs = []
    for b in range(B):
        nme = pool[b % len(pool)]
        L = len(pc.STREAMS[nme]["ranges"])
        recs.append((nme, (b * 7) % (L + 1)))  # prefixes of 0 .. L scans
    o = _odom(pkg, base, B)
    got = o.process([pc.STREAMS[n]["ranges"][:l] for n, l in recs], [pc.STREAMS[n]["stamps"][:l] for n, l in recs])
    o.close()
    for b, (n, l) in enumerate(recs):
        assert _same(got[b], ref[n][:l]), (b, n, l)


@pytest.mark.parametrize("n", [3, 1081, 2408])
def test_beam_counts(pkg, n):
    """The handle runs at 3, 1081 and 2408 beams (the pair kernel's limit on an H100) and equals the restatement."""
    st = dict(pc.STREAMS["straight"])
    r = st["ranges"][:12]
    st["ranges"] = np.ascontiguousarray(np.resize(r, (len(r), n)) if n != 1081 else r)
    st["stamps"] = st["stamps"][:12]
    o = _odom(pkg, st, 1, n)
    got = o.process([st["ranges"]], [st["stamps"]])[0]
    o.close()
    compare(st, got, pc.restate(st), f"n={n}")


def test_too_many_beams_refused(pkg):
    M = pkg.load("matcher")
    with pytest.raises(M.B2SError) as e:
        _odom(pkg, pc.STREAMS["straight"], 4, 2409)
    assert e.value.status == pkg.abi.B2S_ERR_TOO_LARGE
