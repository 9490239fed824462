"""K3 (lesson3 PL-ICP).  Parity with CSM itself is UNPINNED (CSM is external and un-versioned).  What is pinned:

* the CPU restatement (oracle/plicp_oracle.c) against tests/plicp_reference.py, an independent float64 statement of
  ONE iteration written from the paper (its point-to-line solve eliminates t and finds theta with brentq; no quartic).
  Iteration by iteration, from the first guess, from the restatement's own iterates and from perturbed estimates:
  on every step none of whose discrete decisions lies within 1e-9 of flipping (the reference reports the margins),
  `valid` and `nvalid` are equal, x agrees to XTOL = 1e-11 and `error` to 1e-10 relative (not gpu);
* the CUDA kernel against both in the same way, and its whole loop against the restatement's: `valid`, `iterations`
  and `nvalid` exactly unless the reference marks a step of the run borderline, x to XTOL — over a settings matrix,
  geometric edge cases, 3 .. 2 408 beams (the largest count the shared-memory kernel takes on an H100), batches of
  1, 1 024 and 9 999 pairs (gpu);
* recovery of known synthetic transforms to <= 1e-4 on noise-free scans (not gpu and gpu).

The library builds with -fmad=false, so apart from the device's double cos / sin / atan / atan2 (which may differ from
glibc in the last place) the kernel does the restatement's arithmetic: a step that is not borderline has no reason
to differ by more than rounding."""
import ctypes as C

import numpy as np
import pytest

import plicp_reference as ref
from oracle import port

RMIN, RMAX = 0.1, 30.0
XTOL = 1e-11        # |x| difference allowed between two implementations on a step that is not borderline
ERR_RTOL = 1e-10    # relative difference of `error` (a sum over ~1000 distances in another order)
CASES = [(0.05, -0.03, 0.02), (0.2, 0.1, 0.1), (0.0, 0.0, 0.0), (-0.3, 0.25, -0.15), (0.12, -0.4, 0.3)]


def hokuyo_theta(synth):
    laser = synth.Laser()
    return laser, laser.min_angle + np.arange(laser.n_readings) * laser.angular_resolution


def ring(synth, n):
    """a 360-degree lidar of n beams and its beam angles"""
    inc = 2 * np.pi / n
    laser = synth.Laser(n_readings=n, min_angle=-np.pi, max_angle=np.pi - inc, angular_resolution=inc)
    return laser, laser.min_angle + np.arange(n) * inc


def pair(synth, world, d, laser, rng=None, dropout=0.0):
    pa = np.array([0.3, -0.2, 0.4])
    c, s = np.cos(pa[2]), np.sin(pa[2])
    pb = np.array([pa[0] + c * d[0] - s * d[1], pa[1] + s * d[0] + c * d[1], pa[2] + d[2]])
    return synth.cast_scan(world, pa, laser, rng, dropout=dropout), synth.cast_scan(world, pb, laser, rng, dropout=dropout)


def one_step(P):
    return port.abi.icp_params(**{f: getattr(P, f) for f, _ in P._fields_ if f != "max_iterations"}, max_iterations=1)


def close(a, b, tol=XTOL):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() <= tol


def err_close(a, b, atol=1e-13):
    return abs(a - b) <= ERR_RTOL * max(abs(a), abs(b)) + atol


def step_cases(synth, quick=False):
    """(label, P, ref, sens, theta, guesses): several worlds, noise, dropouts, point-to-line and point-to-point, a narrow
    angular window (its edges decide correspondences) and a 360-degree scan (the +-2 pi wrap).  The guesses are the
    first guess (zero, as the odometry's first call, or small), the restatement's own iterates from it up to
    convergence and two perturbations of the truth."""
    abi = port.abi
    laser, theta = hokuyo_theta(synth)
    rlaser, rtheta = ring(synth, 720)
    rng = np.random.default_rng(11)
    params = [("p2l", abi.icp_params()), ("p2p", abi.icp_params(use_point_to_line_distance=0)),
              ("narrow", abi.icp_params(max_angular_correction_deg=0.5, max_linear_correction=0.01)),
              ("p2l-nodoubles", abi.icp_params(outliers_remove_doubles=0, outliers_adaptive_mult=1.5))]
    out = []
    worlds = (10, 11) if quick else (10, 11, 12)
    for w in worlds:
        world = synth.make_world(w)
        for k, d in enumerate((CASES[1], CASES[3], (0.03, 0.02, -0.01))):
            noisy, drop = (w + k) % 2 == 0, 0.05 if k == 1 else 0.0
            lz, th = (rlaser, rtheta) if (w, k) in ((11, 2), (12, 0)) else (laser, theta)
            ra, rb = pair(synth, world, d, lz, rng if noisy else None, drop)
            if k == 2:
                ra[200:260] = np.nan  # a long invalid run: segment ends far apart
                rb[::41] = 0.0
            for pi, (label, P) in enumerate(params[:2] if quick else params):
                x = np.zeros(3) if pi < 2 else np.array([0.01, -0.005, 0.004])
                guesses = [x]
                for _ in range(5):
                    res = port.plicp_match(one_step(P), ra, rb, th, RMIN, RMAX, x)
                    if not res.valid or np.abs(np.array(res.x[:]) - x).max() < 1e-9:
                        break  # past convergence noise-free residuals are rounding: every trimming decision is a toss
                    x = np.array(res.x[:])
                    guesses.append(x)
                guesses += [np.array(d) + [0.02, -0.01, 0.01], np.array(d) * 0.5]
                out.append((f"w{w}/{k}/{label}/n{len(th)}", P, ra, rb, th, guesses))
    return out


def check_step(got, st):
    """got = (valid, nvalid, x, error) of one iteration; st = the reference's Step.  -> max |dx| (0 if not compared)"""
    valid, nvalid, x, error = got
    assert valid == st.valid and nvalid == st.nvalid, (valid, st.valid, nvalid, st.nvalid)
    assert err_close(error, st.error), (error, st.error)
    dx = float(np.abs(np.asarray(x) - st.x).max())
    assert dx <= XTOL, (x, st.x)
    return dx


# ---------------------------------------------------------------- CPU: restatement vs the float64 reference

def test_restatement_matches_reference_step_by_step(pkg):
    synth = pkg.synth
    steps = borderline = 0
    worst = 0.0
    for label, P, ra, rb, th, guesses in step_cases(synth):
        P1 = one_step(P)
        for g in guesses:
            st = ref.step(P1, ra, rb, th, RMIN, RMAX, g)
            res = port.plicp_match(P1, ra, rb, th, RMIN, RMAX, g)
            steps += 1
            if st.borderline:
                borderline += 1
                continue
            assert res.iterations == st.valid, (label, g)
            worst = max(worst, check_step((res.valid, res.nvalid, res.x[:], res.error), st))
    print(f"\nrestatement vs reference: {steps} steps, {borderline} borderline, max |dx| {worst:.2e} (XTOL {XTOL:g})")
    assert steps >= 150 and borderline <= steps // 10


def test_restatement_loop_is_its_single_steps(pkg):
    """the whole loop is the chain of one-iteration calls, bit for bit: what the step tests pin is what the loop does"""
    synth = pkg.synth
    for label, P, ra, rb, th, _ in step_cases(synth, quick=True):
        full = port.plicp_match(P, ra, rb, th, RMIN, RMAX, [0, 0, 0])
        x, nv, it, ok = np.zeros(3), 0, 0, 1
        for it in range(P.max_iterations + 1):
            if it == P.max_iterations:
                break
            r = port.plicp_match(one_step(P), ra, rb, th, RMIN, RMAX, x)
            nv = r.nvalid
            if not r.valid:
                ok = 0
                break
            xn = np.array(r.x[:])
            d = xn - x
            c, s = np.cos(x[2]), np.sin(x[2])
            x = xn
            if np.hypot(c * d[0] + s * d[1], -s * d[0] + c * d[1]) < P.epsilon_xy and abs(d[2]) < P.epsilon_theta:
                it += 1
                break
        assert (full.valid, full.iterations, full.nvalid) == (ok, it, nv), label
        assert np.array_equal(np.array(full.x[:]), x), label


def test_oracle_recovers_known_transform(pkg):
    abi, synth = pkg.abi, pkg.synth
    laser, theta = hokuyo_theta(synth)
    world = synth.make_world(3)
    for d in CASES:
        ra, rb = pair(synth, world, d, laser)
        res = port.plicp_match(abi.icp_params(), ra, rb, theta, RMIN, RMAX, [0, 0, 0])
        assert res.valid == 1 and res.nvalid > 500
        assert np.abs(np.array(res.x[:]) - np.array(d)).max() <= 1e-4
    # noisy scans: centimetre-level recovery; a first guess helps
    rng = np.random.default_rng(0)
    ra, rb = pair(synth, world, CASES[1], laser, rng)
    res = port.plicp_match(abi.icp_params(), ra, rb, theta, RMIN, RMAX, [0.15, 0.05, 0.08])
    assert res.valid == 1 and np.abs(np.array(res.x[:]) - np.array(CASES[1])).max() < 0.02
    # too few valid readings -> invalid (sm_result.valid = 0)
    bad = np.full(1081, 100.0)
    res = port.plicp_match(abi.icp_params(), bad, bad, theta, RMIN, RMAX, [0, 0, 0])
    assert res.valid == 0


def duplicated_beam(synth):
    """a reference scan with one beam repeated (same angle, same range): the segment between the two copies has
    length zero, its normal is 0/0 and the point-to-line solve has no finite solution"""
    laser, theta = hokuyo_theta(synth)
    ra, rb = pair(synth, synth.make_world(3), CASES[0], laser)
    theta = theta.copy()
    theta[501] = theta[500]
    ra[501] = ra[500]
    rb[501] = rb[500]
    return ra, rb, theta


def sparse_pairs(synth):
    """valid readings only at beam 0 / n-1 and a few interior ones: correspondences around the 5 floor.  The first
    pair fails in its second iteration (no correspondence left after a wild first solve) and keeps its first
    estimate; the last fails at once with 4.  Five or six correspondences make an ill-conditioned solve: the float64
    reference's estimate differs from the restatement's by up to 2e-11 here, so these runs are compared to 1e-9"""
    laser, theta = hokuyo_theta(synth)
    n = len(theta)
    ra, rb = pair(synth, synth.make_world(14), CASES[0], laser)
    out = []
    for keep in ([0, n - 1, 150, 151, 152, 450, 451, 452, 800, 801, 802], [0, n - 1, 300, 301, 600, 601, 900, 901],
                 [0, 1, n - 2, n - 1, 200, 201, 500, 501, 502], [0, n - 1, 300, 301, 302, 600, 601, 602, 603]):
        a, b = np.full(n, np.nan), np.full(n, np.inf)
        a[keep], b[keep] = ra[keep], rb[keep]
        out.append((a, b))
    return out


SPARSE_OUTCOMES = dict(valid=[0, 1, 1, 0], iterations=[1, 3, 2, 0], nvalid=[0, 5, 6, 4])


def test_restatement_failures_match_reference(pkg):
    """runs that end in a failed iteration (too few correspondences, at the first or a later iteration; a solve
    without a finite solution): valid, iterations, nvalid and the estimate kept"""
    abi, synth = pkg.abi, pkg.synth
    _, theta = hokuyo_theta(synth)
    P = abi.icp_params()
    got = []
    for a, b in sparse_pairs(synth):
        res = port.plicp_match(P, a, b, theta, RMIN, RMAX, [0, 0, 0])
        rv, rit, rnv, rx, flags = ref.iterate(P, a, b, theta, RMIN, RMAX, [0, 0, 0], XTOL)
        assert not flags and (res.valid, res.iterations, res.nvalid) == (rv, rit, rnv)
        assert close(res.x[:], rx, 1e-9)
        got.append((res.valid, res.iterations, res.nvalid))
    assert [list(g) for g in zip(*got)] == list(SPARSE_OUTCOMES.values())
    for a, b in sparse_pairs(synth):  # the same runs one iteration at a time
        r1 = port.plicp_match(one_step(P), a, b, theta, RMIN, RMAX, [0, 0, 0])
        st = ref.step(one_step(P), a, b, theta, RMIN, RMAX, [0, 0, 0])
        assert (r1.valid, r1.iterations, r1.nvalid) == (st.valid, st.valid, st.nvalid)


def test_failed_solve_keeps_the_last_estimate(pkg):
    abi, synth = pkg.abi, pkg.synth
    ra, rb, theta = duplicated_beam(synth)
    guess = [0.01, -0.02, 0.005]
    res = port.plicp_match(abi.icp_params(), ra, rb, theta, RMIN, RMAX, guess)
    st = ref.step(one_step(abi.icp_params()), ra, rb, theta, RMIN, RMAX, guess)
    assert res.valid == 0 and res.iterations == 0 and res.nvalid >= 5
    assert list(res.x[:]) == guess
    assert st.valid == 0 and st.nvalid == res.nvalid and not st.borderline


def test_argument_checks_and_no_device(pkg):
    abi = pkg.abi
    P, M = pkg.load("plicp"), pkg.load("matcher")
    L = P._bind()
    n, B = 1081, 2
    r, th, g = np.full(B * n, 5.0), np.linspace(-2, 2, n), np.zeros(3 * B)
    out = (abi.IcpResult * B)()
    d = port._d

    def call(params=abi.icp_params(), batch=B, n=n, ref=d(r), sens=d(r), theta=d(th), guess=d(g), res=out):
        return L.b2s_plicp_match(C.byref(params) if params is not None else None, batch, n, ref, sens, theta, RMIN, RMAX,
                                 guess, 0, None, res)

    for kw in (dict(batch=0), dict(batch=-1), dict(n=2), dict(n=0), dict(params=abi.icp_params(max_iterations=0)),
               dict(params=abi.icp_params(max_iterations=-3)), dict(params=None), dict(ref=None), dict(sens=None),
               dict(theta=None), dict(guess=None), dict(res=None)):
        assert call(**kw) == abi.B2S_ERR_BAD_PARAMS, kw
    if M.device_count() > 0:
        return
    assert call() == abi.B2S_ERR_NO_DEVICE  # no CPU fallback


# ---------------------------------------------------------------- device

def device_steps(P_mod, P1, items):
    """items: [(ra, rb, theta, guess)] sharing theta -> (x, valid, iterations, nvalid, error) of one device call"""
    th = items[0][2]
    return P_mod.match(P1, [i[0] for i in items], [i[1] for i in items], th, RMIN, RMAX, [i[3] for i in items])


@pytest.mark.gpu
def test_gpu_matches_reference_step_by_step(pkg):
    synth = pkg.synth
    Pm = pkg.load("plicp")
    steps = borderline = 0
    worst_ref = worst_orc = 0.0
    for label, P, ra, rb, th, guesses in step_cases(synth):
        P1 = one_step(P)
        x, valid, iters, nvalid, err = device_steps(Pm, P1, [(ra, rb, th, g) for g in guesses])
        for b, g in enumerate(guesses):
            st = ref.step(P1, ra, rb, th, RMIN, RMAX, g)
            res = port.plicp_match(P1, ra, rb, th, RMIN, RMAX, g)
            steps += 1
            if st.borderline:
                borderline += 1
                continue
            assert iters[b] == st.valid, (label, b)
            worst_ref = max(worst_ref, check_step((valid[b], nvalid[b], x[b], err[b]), st))
            assert (valid[b], nvalid[b]) == (res.valid, res.nvalid), (label, b)
            worst_orc = max(worst_orc, float(np.abs(x[b] - np.array(res.x[:])).max()))
            assert worst_orc <= XTOL and err_close(err[b], res.error), (label, b, x[b], res.x[:])
    print(f"\ndevice steps: {steps}, {borderline} borderline; max |dx| vs reference {worst_ref:.2e}, "
          f"vs restatement {worst_orc:.2e} (XTOL {XTOL:g})")
    assert steps >= 150 and borderline <= steps // 10


def loop_check(Pm, P, refs, sens, theta, guesses, label="", xtol=XTOL):
    """device whole loop vs the restatement's; exact counts unless the reference marks the run borderline.
    -> (device arrays, restatement results, number of borderline runs)"""
    got = Pm.match(P, refs, sens, theta, RMIN, RMAX, guesses)
    x, valid, iters, nvalid, err = got
    results, nb, exact = [], 0, 0
    for b in range(len(refs)):
        res = port.plicp_match(P, refs[b], sens[b], theta, RMIN, RMAX, guesses[b])
        results.append(res)
        rv, rit, rnv, rx, flags = ref.iterate(P, refs[b], sens[b], theta, RMIN, RMAX, guesses[b], XTOL)
        if flags:
            # A decision of the run lies within rounding of flipping (typically: trimming among the rounding-level
            # residuals of a noise-free pair at its exact solution).  Only here is slack allowed: one correspondence
            # or the iteration at which the stopping test fires may differ; the estimate may not.
            nb += 1
            assert valid[b] == res.valid, (label, b, flags)
            assert abs(int(iters[b]) - res.iterations) <= 1, (label, b, flags)
            if res.error > 1e-6:
                assert abs(int(nvalid[b]) - res.nvalid) <= 3, (label, b, flags)
            if res.valid:
                assert close(x[b], res.x[:], 1e-6), (label, b, flags)
            continue
        exact += 1
        assert (valid[b], iters[b], nvalid[b]) == (res.valid, res.iterations, res.nvalid) == (rv, rit, rnv), \
            (label, b, (valid[b], iters[b], nvalid[b]), (res.valid, res.iterations, res.nvalid), (rv, rit, rnv))
        assert close(x[b], res.x[:], xtol) and close(x[b], rx, xtol), (label, b, x[b], res.x[:], rx)
        # estimates xtol apart move each of the nvalid points by up to xtol times its range (< 30 m)
        assert err_close(err[b], res.error, 30 * xtol * res.nvalid), (label, b, err[b], res.error)
        if not res.iterations:  # a run that failed at once reports its first guess, bit for bit
            assert np.array_equal(x[b], np.asarray(guesses[b], np.float64)), (label, b)
    print(f"\n{label}: {exact} runs exact, {nb} borderline")
    return got, results, nb


@pytest.mark.gpu
def test_gpu_matches_restatement_and_truth(pkg):
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    laser, theta = hokuyo_theta(synth)
    rng = np.random.default_rng(1)
    refs, sens, guesses, truth = [], [], [], []
    for w in range(3):
        world = synth.make_world(10 + w)
        for k, d in enumerate(CASES):
            ra, rb = pair(synth, world, d, laser, rng if k % 2 else None)
            if k == 3:
                ra[100:140] = np.nan  # invalid readings
                rb[::37] = 0.0
            refs.append(ra); sens.append(rb); truth.append(d)
            guesses.append([0, 0, 0] if k % 2 == 0 else list(np.array(d) * 0.7))
    refs.append(np.full(1081, 100.0)); sens.append(np.full(1081, 100.0)); guesses.append([0, 0, 0]); truth.append((0, 0, 0))
    (x, valid, _, _, _), _, nb = loop_check(Pm, abi.icp_params(), refs, sens, theta, guesses, "default")
    for b in (0, 2, 5 + 0, 5 + 2):  # noise-free pairs: truth recovered
        assert valid[b] == 1 and np.abs(x[b] - np.array(truth[b])).max() <= 1e-4
    assert valid[-1] == 0
    # point-to-point and no duplicate pruning through the same kernel
    p2 = abi.icp_params(use_point_to_line_distance=0, outliers_remove_doubles=0, max_iterations=30)
    loop_check(Pm, p2, refs[:5], sens[:5], theta, guesses[:5], "p2p")


@pytest.mark.gpu
def test_gpu_settings_matrix(pkg):
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    laser, theta = hokuyo_theta(synth)
    world = synth.make_world(13)
    rng = np.random.default_rng(3)
    refs, sens = zip(*[pair(synth, world, d, laser, rng if i % 2 else None) for i, d in enumerate(CASES[:4])])
    g0 = [[0, 0, 0], [0.1, 0.05, 0.05], [0.01, -0.01, 0.0], [-0.2, 0.2, -0.1]]

    def run(label, **kw):
        P = abi.icp_params(**kw)
        got, results, _ = loop_check(Pm, P, refs, sens, theta, g0, label)
        return P, got, results

    _, (x, v, it, nv, _), _ = run("eps0", epsilon_xy=0.0, epsilon_theta=0.0)
    assert np.all(v == 1) and np.all(it == 10)
    _, (x, v, it, nv, _), _ = run("one", max_iterations=1)
    assert np.all(v == 1) and np.all(it == 1)
    _, (x, v, it, nv, _), _ = run("huge-eps", epsilon_xy=1e9, epsilon_theta=1e9)
    assert np.all(v == 1) and np.all(it == 1)
    for order in (0.0, 1.0):
        # maxPerc 0 keeps the single nearest correspondence (and exact ties): too few, invalid, x = the first guess
        _, (x, v, it, nv, _), _ = run(f"perc0/{order}", outliers_maxPerc=0.0, outliers_adaptive_order=order,
                                      outliers_adaptive_mult=1e9)
        assert np.all(v == 0) and np.all(it == 0) and np.all(nv < 5) and np.array_equal(x, np.array(g0, np.float64))
        for perc in (1.0, 0.9):
            P, (x, v, it, nv, _), _ = run(f"perc{perc}/{order}", outliers_maxPerc=perc, outliers_adaptive_order=order,
                                          outliers_adaptive_mult=1e9, max_iterations=1)
            for b in range(len(refs)):
                st = ref.step(P, refs[b], sens[b], theta, RMIN, RMAX, g0[b])
                # nothing trimmed at 1.0; at 0.9 the floor(0.9 k) + 1 nearest (no two distances tie)
                assert nv[b] == (st.k if perc == 1.0 else int(np.floor(st.k * perc)) + 1), (perc, order, b, nv[b], st.k)
    run("p2l-nodoubles", outliers_remove_doubles=0)
    _, (x, v, it, nv, e), _ = run("nothing-matches", max_correspondence_dist=1e-9)
    assert np.all(v == 0) and np.all(it == 0) and np.all(nv == 0) and np.all(e == 0)
    assert np.array_equal(x, np.array(g0, np.float64))
    P, _, _ = run("whole-window", max_angular_correction_deg=800.0)
    n = len(theta)
    assert 800.0 * np.pi / 180 / ((theta[-1] - theta[0]) / n) > 2 * n  # every window is clipped to [0, n - 1]


@pytest.mark.gpu
def test_gpu_geometry_edges(pkg):
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    laser, theta = hokuyo_theta(synth)
    n = len(theta)
    world = synth.make_world(14)
    P = abi.icp_params()
    # identical scans: every distance 0, all but the two extremal beams kept, converged at once at ~0
    ra, _ = pair(synth, world, CASES[2], laser)
    (x, v, it, nv, e), res, nb = loop_check(Pm, P, [ra], [ra], theta, [[0, 0, 0]], "identical")
    assert nb == 0 and (v[0], it[0], nv[0], e[0]) == (1, 1, n - 2, 0.0) and np.abs(x[0]).max() < 1e-12
    # valid readings only at beam 0 / n-1 and a few interior ones (see sparse_pairs)
    sparse = sparse_pairs(synth)
    (x, v, it, nv, e), res, nb = loop_check(Pm, P, [s[0] for s in sparse], [s[1] for s in sparse], theta,
                                            [[0, 0, 0]] * 4, "sparse", xtol=1e-9)
    assert nb == 0 and [list(v), list(it), list(nv)] == list(SPARSE_OUTCOMES.values())
    assert np.abs(x[0]).max() > 1.0 and np.array_equal(x[3], np.zeros(3))
    # long invalid runs and every kind of invalid reading: exactly range_min / range_max, 0, negative, inf, NaN
    ra, rb = pair(synth, world, CASES[1], laser, np.random.default_rng(4))
    ra[100:400] = np.nan
    rb[600:750] = np.inf
    for arr, off in ((ra, 0), (rb, 3)):
        arr[410 + off::60] = RMIN
        arr[420 + off::60] = RMAX
        arr[430 + off::60] = 0.0
        arr[440 + off::60] = -2.0
        arr[450 + off::60] = np.inf
        arr[460 + off::60] = np.nan
    _, _, nb = loop_check(Pm, P, [ra], [rb], theta, [[0.15, 0.05, 0.07]], "invalid")
    assert nb == 0
    # a corridor: two long parallel walls, noisy.  Cross-track and heading are observable, along-track is not
    corridor = synth.World(np.array([[-200.0, -1.2, 200.0, -1.2], [-200.0, 1.5, 200.0, 1.5]]), 200.0, 2.0)
    rng = np.random.default_rng(6)
    truth = np.array([0.3, 0.05, 0.03])
    pa = np.array([0.0, 0.0, 0.0])
    ca = synth.cast_scan(corridor, pa, laser, rng)
    cb = synth.cast_scan(corridor, truth, laser, rng)
    (x, v, _, _, _), _, nb = loop_check(Pm, abi.icp_params(max_iterations=30), [ca], [cb], theta, [[0, 0, 0]],
                                        "corridor")
    assert v[0] == 1  # (the zero first guess puts the last beam on the +-2 pi wrap: the run may be borderline)
    assert abs(x[0][1] - truth[1]) < 0.01 and abs(x[0][2] - truth[2]) < 0.005, x[0]


@pytest.mark.gpu
def test_gpu_failed_solve_matches_restatement(pkg):
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    ra, rb, theta = duplicated_beam(synth)
    guess = [[0.01, -0.02, 0.005], [0, 0, 0]]
    for P in (abi.icp_params(), abi.icp_params(max_iterations=1)):
        x, v, it, nv, e = Pm.match(P, [ra, ra], [rb, rb], theta, RMIN, RMAX, guess)
        for b in range(2):
            res = port.plicp_match(P, ra, rb, theta, RMIN, RMAX, guess[b])
            assert (v[b], it[b], nv[b]) == (res.valid, res.iterations, res.nvalid) == (0, 0, res.nvalid)
            assert np.array_equal(x[b], np.array(guess[b], np.float64)) and list(res.x[:]) == guess[b]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 4, 5, 90, 360, 598, 720, 1440, 2000])
def test_gpu_beam_counts_between_the_shared_memory_defaults(pkg, n):
    """Tiny scans, beam counts whose static + dynamic shared memory crosses the 48 KB default without the dynamic
    part alone doing so (86..598 once failed with cudaErrorInvalidValue), and beyond: every count must work like the
    1081-beam lidar and give the restatement's answer."""
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    laser, theta = ring(synth, n)
    world = synth.make_world(4)
    refs, sens = zip(*[pair(synth, world, d, laser) for d in CASES[:3]])
    _, results, nb = loop_check(Pm, abi.icp_params(), refs, sens, theta, [[0, 0, 0]] * 3, f"n={n}")
    if n <= 5:
        assert not any(r.valid for r in results)  # at most 3 usable correspondences
    elif n >= 360:
        assert all(r.valid for r in results)


@pytest.mark.gpu
def test_gpu_wide_scans_and_the_shared_memory_limit(pkg):
    """1440 / 2000-beam 270-degree scans and 360-degree scans of 1081 / 2000 beams against the restatement; then the
    largest beam count the kernel takes (TOO_LARGE is returned before any launch), found by bisection: it must run and
    match, one more beam must be refused"""
    abi, synth = pkg.abi, pkg.synth
    Pm, M = pkg.load("plicp"), pkg.load("matcher")
    world = synth.make_world(5)
    P = abi.icp_params()
    for n, full in ((1440, False), (2000, False), (1081, True), (2000, True)):
        if full:
            laser, theta = ring(synth, n)
        else:
            inc = np.deg2rad(270.0) / (n - 1)
            laser = synth.Laser(n_readings=n, angular_resolution=inc, max_angle=synth.Laser().min_angle + (n - 1) * inc)
            theta = laser.min_angle + np.arange(n) * inc
        refs, sens = zip(*[pair(synth, world, d, laser, np.random.default_rng(n)) for d in CASES[:2]])
        _, results, nb = loop_check(Pm, P, refs, sens, theta, [[0, 0, 0]] * 2, f"n={n}/{full}")
        assert all(r.valid for r in results)

    def fits(n):
        _, th = ring(synth, n)
        try:
            Pm.match(P, np.full((1, n), 5.0), np.full((1, n), 5.0), th, RMIN, RMAX, [[0, 0, 0]])
            return True
        except M.B2SError as e:
            assert e.status == abi.B2S_ERR_TOO_LARGE, e
            return False

    lo, hi = 2000, 65536
    assert fits(lo) and not fits(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    print(f"\nlargest PL-ICP beam count: {lo}")
    laser, theta = ring(synth, lo)
    refs, sens = zip(*[pair(synth, world, d, laser) for d in CASES[:2]])
    _, results, nb = loop_check(Pm, P, refs, sens, theta, [[0, 0, 0]] * 2, f"n={lo}")
    assert all(r.valid for r in results)
    assert not fits(lo + 1)


def bit_equal(a, b):
    return all(np.array_equal(np.asarray(p).view(np.uint8), np.asarray(q).view(np.uint8)) for p, q in zip(a, b))


@pytest.mark.gpu
def test_gpu_batch_shapes(pkg):
    """batch 1, the 1 024-pair batch and the 9 999-pair odometry batch bench.py runs: a pair's result does not depend
    on its position in the batch or on its neighbours (sampled pairs, the first and last included, bit-identical to
    the same pairs run alone or in a small batch), and sampled pairs match the restatement"""
    abi, synth = pkg.abi, pkg.synth
    Pm = pkg.load("plicp")
    laser, theta = hokuyo_theta(synth)
    P = abi.icp_params()
    # 1 024 independent pairs, the bench's recipe
    rng = np.random.default_rng(5)
    world = synth.make_world(33)
    refs, sens = [], []
    for _ in range(64):
        pa = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-np.pi, np.pi)])
        d = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05)])
        c, s = np.cos(pa[2]), np.sin(pa[2])
        pb = np.array([pa[0] + c * d[0] - s * d[1], pa[1] + s * d[0] + c * d[1], pa[2] + d[2]])
        refs.append(synth.cast_scan(world, pa, laser, rng)); sens.append(synth.cast_scan(world, pb, laser, rng))
    refs, sens = np.tile(np.stack(refs), (16, 1)), np.tile(np.stack(sens), (16, 1))
    guess = np.zeros((1024, 3))
    guess[1::3] = [0.02, -0.01, 0.01]
    big = Pm.match(P, refs, sens, theta, RMIN, RMAX, guess)
    for b in (0, 1, 63, 64, 517, 1022, 1023):
        one = Pm.match(P, refs[b:b + 1], sens[b:b + 1], theta, RMIN, RMAX, guess[b:b + 1])
        assert bit_equal([a[b:b + 1] for a in big], one), b
    small = Pm.match(P, refs[1020:], sens[1020:], theta, RMIN, RMAX, guess[1020:])
    assert bit_equal([a[1020:] for a in big], small)
    for b in range(64):  # tiled copies with the same guess are the same pair
        same = [b + 64 * k for k in range(16) if (b + 64 * k) % 3 == b % 3]
        for a in big:
            assert np.all(a[same] == a[same[0]]), b
    loop_check(Pm, P, refs[[0, 1, 2, 1023]], sens[[0, 1, 2, 1023]], theta, guess[[0, 1, 2, 1023]], "bench")
    # 9 999 consecutive pairs of one 10 000-scan recording (the bench's odometry stream)
    _, _, r = synth.make_trajectory(22, 10000, laser, step_xy=0.05, step_th_deg=1.0)
    g = np.zeros((9999, 3))
    big = Pm.match(P, r[:-1], r[1:], theta, RMIN, RMAX, g)
    assert big[1].sum() >= 9900
    for lo, hi in ((0, 4), (4997, 5003), (9995, 9999)):
        small = Pm.match(P, r[lo:hi], r[lo + 1:hi + 1], theta, RMIN, RMAX, g[lo:hi])
        assert bit_equal([a[lo:hi] for a in big], small), lo
    one = Pm.match(P, r[9998:9999], r[9999:], theta, RMIN, RMAX, g[:1])
    assert bit_equal([a[9998:] for a in big], one)
    idx = [0, 1, 5000, 9997, 9998]
    loop_check(Pm, P, r[idx], r[[i + 1 for i in idx]], theta, g[idx], "stream")
