"""lesson3's odometry node fleet on the device (b2s_plicp_odom_create_fleet / _process_fleet): every recording with its
own laser, mount, parameters and per-scan range fields, in one handle and one launch, against the restatement (pinned
to the unmodified node by test_plicp_odometry_fleet_reference.py), against single-recording handles and the uniform
handle byte for byte, and against the library's own pair matcher.

The continuous-output tolerance and the borderline exemption are test_gpu_plicp_odometry.py's (1e-9)."""
import ctypes as C

import numpy as np
import pytest

import plicp_odometry_cases as pc
import plicp_odometry_fleet_cases as fc
import plicp_reference as pr

pytestmark = pytest.mark.gpu
TOL = 1e-9
DISCRETE = ("valid", "iterations", "nvalid", "published", "keyframe", "reference_scan")
CONT = ("position", "orientation", "linear", "angular", "first_guess", "x", "error")
ALL = fc.all_streams()
NAMES = sorted(ALL)


def _theta(las):
    n, amin, ainc = las
    return (np.float32(amin) + np.arange(n, dtype=np.float32) * np.float32(ainc)).astype(np.float64)


def _fleet(pkg, names):
    P = pkg.load("plicp")
    sts = [ALL[n] for n in names]
    return P.Odometry.fleet([fc.odom_params(s) for s in sts], [s["laser"][0] for s in sts],
                            [s["laser"][1] for s in sts], [s["laser"][2] for s in sts])


def _run(o, names, lo=None, hi=None):
    sl = [slice(lo[b] if lo else 0, hi[b] if hi else None) for b in range(len(names))]
    return o.process([ALL[n]["ranges"][sl[b]] for b, n in enumerate(names)],
                     [ALL[n]["stamps"][sl[b]] for b, n in enumerate(names)],
                     [ALL[n]["limits"][sl[b]] for b, n in enumerate(names)])


def _same(a, b):
    return a.tobytes() == b.tobytes()


def compare(st, got, want, name):
    """test_gpu_plicp_odometry.compare on a stream of its own laser and fields: discrete outputs equal and continuous
    ones within TOL up to the first scan the float64 reference flags as borderline."""
    m = fc.masked(st).astype(np.float64)
    for k in range(len(want)):
        if any(got[k][f] != want[k][f] for f in DISCRETE):
            kf = want[k]["reference_scan"]
            flags = pr.iterate(fc.odom_params(st).icp, m[kf], m[k], _theta(st["laser"]), -np.inf, np.inf,
                               want[k]["first_guess"], 1e-9)[4]
            assert flags, f"{name} scan {k}: {[(f, got[k][f], want[k][f]) for f in DISCRETE]} with no borderline decision"
            return k
        for f in CONT:
            a, b = np.asarray(got[k][f], np.float64), np.asarray(want[k][f], np.float64)
            ok = np.isclose(a, b, rtol=0, atol=TOL, equal_nan=True) | (a == b)
            assert ok.all(), f"{name} scan {k} {f}: {a} vs {b}"
    return len(want)


@pytest.fixture(scope="module")
def mixed(pkg):
    """Every old and new stream in ONE fleet handle, one call."""
    o = _fleet(pkg, NAMES)
    out = dict(zip(NAMES, _run(o, NAMES)))
    o.close()
    return out


@pytest.fixture(scope="module")
def alone(pkg):
    """Every stream on a batch = 1 fleet handle of its own."""
    out = {}
    for n in NAMES:
        o = _fleet(pkg, [n])
        out[n] = _run(o, [n])[0]
        o.close()
    return out


@pytest.mark.parametrize("name", NAMES)
def test_mixed_fleet_equals_restatement_and_single(mixed, alone, name):
    """Each recording of the mixed fleet equals the restatement (only the noise-free stop-and-go stream may reach a
    borderline match) and its own batch = 1 handle byte for byte."""
    st = ALL[name]
    upto = compare(st, mixed[name], fc.restate(st), name)
    assert upto == len(st["ranges"]) or name == "stop_and_go", f"{name}: borderline at scan {upto}"
    assert _same(mixed[name], alone[name]), name


def test_equal_fleet_equals_uniform_handle(pkg):
    """B copies of one row with constant range fields through process_fleet equal b2s_plicp_odom_create +
    b2s_plicp_odom_process byte for byte, and so does create + process_fleet."""
    P = pkg.load("plicp")
    names = ["straight", "backward", "jitter_stamps", "equal_stamps", "no_valid_reading"]
    base = pc.STREAMS["straight"]
    recs = [pc.STREAMS[n] for n in names]
    lim = [np.tile(pc.FIELDS[2:4], (len(s["ranges"]), 1)) for s in recs]
    u = P.Odometry(pc.odom_params(base), len(names), 1081, *map(float, pc.FIELDS))
    want = u.process([s["ranges"] for s in recs], [s["stamps"] for s in recs])
    u.reset()
    got_u = u.process([s["ranges"] for s in recs], [s["stamps"] for s in recs], lim)
    u.close()
    f = P.Odometry.fleet([pc.odom_params(base)] * len(names), [1081] * len(names), [pc.FIELDS[0]] * len(names),
                         [pc.FIELDS[1]] * len(names))
    got_f = f.process([s["ranges"] for s in recs], [s["stamps"] for s in recs], lim)
    f.close()
    for b, n in enumerate(names):
        assert _same(got_f[b], want[b]) and _same(got_u[b], want[b]), n


def test_chunking_and_reset(pkg, mixed):
    """Halves, uneven cuts and one scan per call (other recordings idle in some calls), and a cut right after a
    promotion whose fields differ from the next scan's, give the same bytes as one call; reset(b) mid-stream restarts
    only recording b."""
    B, L = len(NAMES), [len(ALL[n]["ranges"]) for n in NAMES]
    o = _fleet(pkg, NAMES)
    fap = NAMES.index("fields_after_promotion")
    assert mixed["fields_after_promotion"]["keyframe"][4] and \
        (ALL["fields_after_promotion"]["limits"][5] != ALL["fields_after_promotion"]["limits"][4]).any()

    def run(cuts):
        o.reset()
        parts = [[] for _ in range(B)]
        for c in range(len(cuts[0]) - 1):
            res = _run(o, NAMES, [cuts[b][c] for b in range(B)], [cuts[b][c + 1] for b in range(B)])
            for b in range(B):
                parts[b].append(res[b])
        return [np.concatenate(p) for p in parts]

    after_promotion = [[0, 5, l] if b == fap else [0, l // 3, l] for b, l in enumerate(L)]
    for cuts in ([[0, l // 2, l] for l in L],
                 [[0, min(3, l), min(3, l) + (b % 4), l] for b, l in enumerate(L)],
                 [[0] + [min(k, l) for k in range(1, max(L) + 1)] for l in L],
                 [[0] + [min(max(0, k - b), l) for k in range(1, max(L) + B + 1)] for b, l in enumerate(L)],
                 after_promotion):
        got = run(cuts)
        for b, n in enumerate(NAMES):
            assert _same(got[b], mixed[n]), (n, cuts[b])
    o.reset()
    first = _run(o, NAMES, None, [5] * B)
    r = NAMES.index("keyframe_fields")
    o.reset(r)
    rest = _run(o, NAMES, [0 if b == r else 5 for b in range(B)], None)
    for b, n in enumerate(NAMES):
        got = rest[b] if b == r else np.concatenate([first[b], rest[b]])
        assert _same(got, mixed[n]), n
    o.close()


@pytest.mark.parametrize("name", NAMES)
def test_each_scan_is_the_pair_matcher(pkg, mixed, name):
    """b2s_plicp_match on the key frame's and the scan's readings, NaN-masked by their own fields, with limits
    (-inf, inf), the recording's theta and the reported first guess returns the reported sm_icp result bit for bit."""
    P = pkg.load("plicp")
    st, got = ALL[name], mixed[name]
    ks = [k for k in range(len(got)) if got[k]["published"]]
    m = fc.masked(st).astype(np.float64)
    x, valid, it, nv, err = P.match(fc.odom_params(st).icp, m[[got[k]["reference_scan"] for k in ks]], m[ks],
                                    _theta(st["laser"]), -np.inf, np.inf, np.stack([got[k]["first_guess"] for k in ks]))
    g = got[ks]
    assert np.array_equal(x.view(np.int64), g["x"].view(np.int64))
    assert np.array_equal(err.view(np.int64), g["error"].view(np.int64))
    assert (valid == g["valid"]).all() and (it == g["iterations"]).all() and (nv == g["nvalid"]).all()


@pytest.mark.parametrize("B", [7, 133, 1000])
def test_ragged_fleets_equal_single_handles(pkg, alone, B):
    """B recordings, prefixes of 0 .. L scans of every stream (3 to 2408 beams), in one call: each equals its own
    batch = 1 handle byte for byte."""
    names = [NAMES[(b * 5) % len(NAMES)] for b in range(B)]
    cnt = [(b * 7) % (len(ALL[n]["ranges"]) + 1) for b, n in enumerate(names)]
    o = _fleet(pkg, names)
    got = _run(o, names, None, cnt)
    o.close()
    for b, n in enumerate(names):
        assert _same(got[b], alone[n][:cnt[b]]), (b, n, cnt[b])


def test_refusals(pkg, alone):
    """A 2409-beam recording in a fleet is refused with TOO_LARGE; a refused process_fleet writes nothing and leaves
    every recording as it was; process on a fleet handle is refused."""
    P, M, abi = pkg.load("plicp"), pkg.load("matcher"), pkg.abi
    with pytest.raises(M.B2SError) as e:
        P.Odometry.fleet([abi.plicp_odom_params()] * 3, [360, 2409, 1081], [-3.1] * 3, [0.01] * 3)
    assert e.value.status == abi.B2S_ERR_TOO_LARGE and "recording 1" in str(e.value)
    names = ["laser_720_360", "fields_after_promotion"]
    o = _fleet(pkg, names)
    first = _run(o, names, None, [3, 3])
    L = P._bind()
    ip, fp, up = C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_uint32)
    out = (abi.PlicpOdomStep * 8)()
    C.memset(out, 0x5A, C.sizeof(out))
    before = bytes(out)
    r = np.zeros(4 * 2408, np.float32)
    lm = np.zeros(16, np.float32)
    sm = np.zeros(16, np.uint32)
    a = (r.ctypes.data_as(fp), lm.ctypes.data_as(fp), sm.ctypes.data_as(up))
    for counts, arrs, status in (([2, -1], a, abi.B2S_ERR_BAD_PARAMS),
                                 ([1, 1], (a[0], None, a[2]), abi.B2S_ERR_BAD_PARAMS),
                                 ([1, 1], (None, a[1], a[2]), abi.B2S_ERR_BAD_PARAMS),
                                 ([1, 1], (a[0], a[1], None), abi.B2S_ERR_BAD_PARAMS),
                                 ([2 ** 31 - 1, 1], a, abi.B2S_ERR_TOO_LARGE)):
        n = np.array(counts, np.int32)
        assert L.b2s_plicp_odom_process_fleet(o._h, n.ctypes.data_as(ip), *arrs, out) == status, counts
        assert bytes(out) == before, counts
    assert L.b2s_plicp_odom_process_fleet(o._h, None, *a, out) == abi.B2S_ERR_BAD_PARAMS
    n = np.array([1, 1], np.int32)
    assert L.b2s_plicp_odom_process(o._h, n.ctypes.data_as(ip), a[0], a[2], out) == abi.B2S_ERR_BAD_PARAMS
    assert bytes(out) == before
    with pytest.raises(ValueError):
        o.process([ALL[n]["ranges"][3:] for n in names], [ALL[n]["stamps"][3:] for n in names])
    rest = _run(o, names, [3, 3], None)
    for b, nme in enumerate(names):
        assert _same(np.concatenate([first[b], rest[b]]), alone[nme]), nme
    o.close()
