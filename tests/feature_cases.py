"""Seeded LaserScans for lesson1's corner picker (b2s_feature_detect, feature_detection.cc:77-179).  The file name keeps
pytest from collecting it; tests import it.

Every family returns float32 [batch][n].  `killer_scans()` reads tests/golden/feature_killer.npz, made by
`python tests/feature_cases.py --write-killer` (solve_killer_scan); the least-squares solve behind it is not
bit-reproducible across BLAS builds, so its result is kept rather than recomputed."""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
synth = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.synth")
KILLER = os.path.join(HERE, "golden", "feature_killer.npz")
MAX_BEAMS = 1500


def _dropouts(r, rng, p=0.02):
    m = rng.random(r.shape)
    r[m < p / 3] = np.nan
    r[(m >= p / 3) & (m < 2 * p / 3)] = np.inf
    r[(m >= 2 * p / 3) & (m < p)] = -np.inf
    return r


def rooms(seed, batch, laser=None, dropout=0.02):
    """synthetic rooms (synth.make_trajectory) with NaN / +inf / -inf dropouts"""
    laser = laser or synth.Laser()
    _, _, r = synth.make_trajectory(seed, batch, laser, step_xy=0.05, step_th_deg=1.0)
    return _dropouts(r.astype(np.float32), np.random.default_rng(seed), dropout)


def quantised(seed, batch, step):
    """room scans rounded to `step` metres (0.001: millimetre, 0.01: centimetre sensors)"""
    r = rooms(seed, batch)
    return (np.round(r.astype(np.float64) / step) * step).astype(np.float32)


def tie_heavy(seed, batch, n=1081):
    """2-8 range levels in runs: the curvature takes few values, so sector cuts are tied"""
    rng = np.random.default_rng(seed)
    out = np.empty((batch, n), np.float32)
    for b in range(batch):
        levels = rng.choice(np.arange(1, 41) * 0.25, size=rng.integers(2, 9), replace=False)
        row, i = [], 0
        while i < n:
            run = int(rng.integers(1, 12))
            row += [levels[rng.integers(len(levels))]] * run
            i += run
        out[b] = np.array(row[:n], np.float32)
    return _dropouts(out, rng, 0.01)


def short_scans(seed):
    """every count of finite readings 0 .. 40 (so every count mod 6), each with a few non-finite readings mixed in;
    one batch per count, [(count, ranges [4][n])]"""
    rng = np.random.default_rng(seed)
    cases = []
    for count in range(41):
        n = count + 3
        rows = []
        for _ in range(4):
            r = rng.uniform(0.5, 3.0, n).astype(np.float32)
            bad = rng.choice(n, 3, replace=False)
            r[bad] = np.array([np.nan, np.inf, -np.inf], np.float32)
            rows.append(r)
        cases.append((count, np.stack(rows)))
    return cases


def full_width(seed, batch):
    """n = 1500, the node's largest scan"""
    laser = synth.Laser(n_readings=MAX_BEAMS, min_angle=-np.pi, max_angle=np.pi - 2 * np.pi / MAX_BEAMS,
                        angular_resolution=2 * np.pi / MAX_BEAMS)
    return rooms(seed, batch, laser)


def signed(seed, batch, n=720):
    """zero and negative ranges (valid for the node: range_min / range_max are not consulted)"""
    rng = np.random.default_rng(seed)
    r = rng.uniform(-3.0, 3.0, (batch, n)).astype(np.float32)
    r[rng.random(r.shape) < 0.1] = 0.0
    r[rng.random(r.shape) < 0.05] = -0.0
    return r


def huge(seed, batch, n=720):
    """finite ranges up to 1e30: the stencil does not overflow, but d * d does (c = inf, tied at the top)"""
    rng = np.random.default_rng(seed)
    r = rng.uniform(0.5, 5.0, (batch, n)).astype(np.float32)
    m = rng.random(r.shape) < 0.02
    r[m] = (10.0 ** rng.uniform(10, 30, m.sum()) * rng.choice([-1, 1], m.sum())).astype(np.float32)
    return r


def nan_curvature(seed, batch, n=360):
    """finite ranges of 3e38: the stencil's partial sum reaches +inf and then subtracts inf, so c is NaN"""
    rng = np.random.default_rng(seed)
    r = rng.uniform(0.5, 5.0, (batch, n)).astype(np.float32)
    for b in range(batch):
        at = int(rng.integers(20, n - 40))
        r[b, at:at + 12] = np.float32(3e38)
    return r


def solve_killer_scan(sector, huge_at=(), seed=0, n=MAX_BEAMS):
    """A scan of n finite readings whose sector `sector` drives std::sort into its heap-sort fallback.
    The wanted order comes from McIlroy's adversary run against the host's std::sort (oracle.features_port).  The
    stencil is solved for it: curvature c_i = d_i^2 with d_i = +-sqrt(wanted c_i), alternating in sign (the stencil is
    well conditioned there), by least squares, and the solution is rounded to float.  The sector's values are 2 + 0.05
    rank apart, so only their order has to survive the rounding.  Readings of 1e20 at sector offsets `huge_at` make
    the 11 curvatures around each infinite: equal maxima, fixed before the adversary runs, which tie the sector's cut
    when there are more than 20 of them."""
    from oracle import features_port as fp
    s, e = n * sector // 6, n * (sector + 1) // 6 - 1
    L = e - s
    huge_beams = [s + p for p in huge_at]
    top = np.zeros(L, bool)
    for h in huge_beams:
        top[h - 5 - s:h + 6 - s] = True
    order = fp.killer_order(L, top)
    c = np.random.default_rng(seed).uniform(0.0, 4.0, n)
    c[s:e] = 2.0 + order * 0.05
    c[e] = 0.25  # S[e] is walked first and unsorted: keep it below the threshold
    rows = [i for i in range(5, n - 5) if all(abs(i - h) > 5 for h in huge_beams)]
    cols = [k for k in range(n) if k not in huge_beams]
    A = np.zeros((len(rows), n))
    for r, i in enumerate(rows):
        A[r, i - 5:i + 6] = 1.0
        A[r, i] = -10.0
    d = np.array([(1.0 if i % 2 == 0 else -1.0) * np.sqrt(c[i]) for i in rows])
    x, *_ = np.linalg.lstsq(A[:, cols], d, rcond=None)
    v = np.zeros(n)
    v[cols] = x + 5.0  # constants are in the stencil's null space
    v[huge_beams] = 1e20
    return v.astype(np.float32)


KILLER_SPECS = [  # (sector, huge_at): tied cut in the killed sector, and one untied
    (2, (20, 200)),
    (4, (60, 180)),
    (1, ()),
]


def killer_scans():
    """[3][1500]: KILLER_SPECS[k] solved; the first two have a tied cut in the killed sector, the last does not"""
    with np.load(KILLER) as z:
        return z["scans"].copy()


if __name__ == "__main__":
    if "--write-killer" in sys.argv:
        scans = np.stack([solve_killer_scan(s, h, seed=k) for k, (s, h) in enumerate(KILLER_SPECS)])
        np.savez_compressed(KILLER, scans=scans)
        print(KILLER, scans.shape)
