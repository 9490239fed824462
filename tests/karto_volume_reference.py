"""Crafted inputs for the Karto correlative matcher's kernel paths that scans of real rooms never reach, and an
independent reference of its integer response volume.

`brute_volume` computes the volume straight from the flat-index definition of GetResponse's numerator
(Mapper.cpp:819-856):

    sums[y][x][k] = SUM_i grid[base00 + lut[k, i] + stride * (y * width_step + x)]

where a position outside [0, data_size) counts 0 and INT32_MAX marks an invalid reading.  It is numpy gathers and
shares no code with oracle/karto_oracle.c.  Everything after the integer volume (responses, penalties, ties, pose,
covariance) is checked against the C restatement, which `Batch.oracle` runs on the same crafted grid.

The builders below make the cases tests/test_gpu_matcher_edges.py runs on the device.  The tests in this file run
without a GPU: each checks that brute_volume and the restatement agree on a case, and that the case still reaches the
edge it exists for (a class of more than 512 beams, a rounding-tie centre, exactly 512 ties, ...).  A case that
drifts away from its edge then fails here.  The file name is not a test_ name, so run it by name:
`pytest tests/karto_volume_reference.py`.
"""
import importlib
import math

import numpy as np
import pytest

from oracle import port

PKG = "creating-2d-laser-slam-from-scratch_b200"
abi = importlib.import_module(PKG + ".abi")
synth = importlib.import_module(PKG + ".synth")

D = abi.KT_PI_180
INVALID_SCAN = np.iinfo(np.int32).max
GRID_OCCUPIED = 100

# H100 numbers the cases are sized against: cudaDeviceProp::sharedMemPerBlockOptin, and the largest beam count the
# window kernel's list stage takes (n * 26 + 64 <= 200 KB, karto_sweep_plan.cuh)
SMEM_OPTIN = 232_448
LIST_MAX_BEAMS = 7_874
WIN_FLUSH_BEAMS = 512     # beams between flushes of the window kernel's packed-u16 accumulators
RED_MAX_TIES = 512        # k_reduce sums at most this many ties sequentially in reference order
RED_THREADS = 512


# ------------------------------------------------------------------------------------------------ the references

def kround(v):
    """math::Round (Math.h:87-90): half away from zero."""
    v = np.asarray(v, dtype=np.float64)
    return np.where(v >= 0.0, np.floor(v + 0.5), np.ceil(v - 0.5))


def volume_at(grid, lut, bases, data_size):
    """int64 [len(bases)][nA]: SUM_i grid[bases[c] + lut[k, i]] over valid readings, 0 outside [0, data_size)."""
    g = np.asarray(grid).astype(np.int64)
    b = np.asarray(bases, dtype=np.int64).reshape(-1, 1)
    out = np.zeros((b.shape[0], lut.shape[0]), dtype=np.int64)
    for k in range(lut.shape[0]):
        o = lut[k][lut[k] != INVALID_SCAN].astype(np.int64)
        idx = b + o[None, :]
        inside = (idx >= 0) & (idx < data_size)
        out[:, k] = np.where(inside, g[np.clip(idx, 0, data_size - 1)], 0).sum(axis=1)
    return out


def brute_volume(grid, lut, base00, width_step, data_size, nx, ny, stride):
    """int64 sums[y][x][theta] of a regular candidate lattice with its first candidate at flat index base00."""
    iy, ix = np.meshgrid(np.arange(ny, dtype=np.int64), np.arange(nx, dtype=np.int64), indexing="ij")
    bases = int(base00) + stride * (iy * width_step + ix)
    return volume_at(grid, lut, bases.ravel(), data_size).reshape(ny, nx, lut.shape[0])


def lattice(center, grid_off, search, g, resolution):
    """Grid cells (gx, gy) [ny][nx] of CorrelateScan's candidates (Mapper.cpp:338-358, CorrelationGrid::GridIndex),
    as k_bases forms them: kround(((cx + x) - gox) * scale) + roi."""
    scale = 1.0 / resolution
    nx, ny = abi.n_steps(search.offset_x, search.res_x), abi.n_steps(search.offset_y, search.res_y)
    x = -search.offset_x + np.arange(nx, dtype=np.float64) * search.res_x
    y = -search.offset_y + np.arange(ny, dtype=np.float64) * search.res_y
    gx = kround(((center[0] + x) - grid_off[0]) * scale).astype(np.int64) + g.roi_x
    gy = kround(((center[1] + y) - grid_off[1]) * scale).astype(np.int64) + g.roi_y
    return np.broadcast_to(gx[None, :], (ny, nx)), np.broadcast_to(gy[:, None], (ny, nx))


def is_regular(gx, gy, stride):
    ny, nx = gx.shape
    return bool((gx == gx[0, 0] + stride * np.arange(nx)[None, :]).all() and
                (gy == gy[0, 0] + stride * np.arange(ny)[:, None]).all())


def covers(origins, p, width_step, nx, ny, stride):
    """whether flat index p is a cell of the window at each origin: p = a + stride * (iy * width_step + ix)"""
    d = p - np.asarray(origins, dtype=np.int64)
    q = d // stride
    return (d >= 0) & (d % stride == 0) & (q // width_step < ny) & (q % width_step < nx)


def search_stride(search, resolution):
    r = 1.0 / (1.0 / resolution)
    return 1 if search.res_x == r else 2


# ------------------------------------------------------------------------------------------------ cases

def make_laser(n, span_deg=270.0, rt=9.25):
    return synth.Laser(n_readings=n, min_angle=synth.deg2rad(-span_deg / 2), angular_resolution=synth.deg2rad(span_deg / n),
                       range_threshold=rt)


class Batch:
    """B matches of one matcher geometry: scans, crafted grids and their offsets, search centres.  The same arrays go to
    the device handle (set_scans + set_grids) and, one match at a time, to the restatement."""

    def __init__(self, params, laser_s, ranges, poses):
        self.params, self.laser_s, self.laser = params, laser_s, abi.laser_from(laser_s)
        self.ranges = np.ascontiguousarray(ranges, dtype=np.float64)
        self.poses = np.ascontiguousarray(poses, dtype=np.float64)
        self.B = len(self.poses)
        self.pms = []
        for b in range(self.B):
            pm = port.PortMatcher(params, self.laser)
            pm.set_scan(self.ranges[b], self.poses[b])
            self.pms.append(pm)
        self.g = self.pms[0].g
        self.resolution = 1.0 / (1.0 / params.resolution)
        r = self.resolution
        # the grid offset that centres the ROI on the scan (Mapper.cpp:212-220)
        self.offs = np.array([[pm.sp[0] - (0.5 * (self.g.roi_w - 1) * r), pm.sp[1] - (0.5 * (self.g.roi_h - 1) * r)]
                              for pm in self.pms])
        self.grids = np.zeros((self.B, self.g.data_size), dtype=np.uint8)
        self.centers = np.stack([pm.sp for pm in self.pms])

    def _pm(self, b):
        pm = self.pms[b]
        pm.grid = np.ascontiguousarray(self.grids[b])
        pm.grid_off = np.ascontiguousarray(self.offs[b], dtype=np.float64)
        return pm

    def lut(self, b, search):
        return self._pm(b).compute_offsets(self.centers[b][2], search.angle_offset, search.angle_res)

    def oracle(self, b, search, cov_in=None):
        """-> (status, MatchResult, int32 sums [ny][nx][nA]) of the restatement"""
        pm = self._pm(b)
        rc, res = pm.correlate_scan(self.centers[b], search, cov_in=cov_in, want_sums=True)
        return rc, res, pm.last_sums

    def cells(self, b, search):
        return lattice(self.centers[b], self.offs[b], search, self.g, self.resolution)

    def brute(self, b, search):
        """brute_volume of match b (any lattice: irregular ones are summed at their own bases)"""
        gx, gy = self.cells(b, search)
        lut = self.lut(b, search)
        ws, ds = self.g.width_step, self.g.data_size
        stride = search_stride(search, self.resolution)
        if is_regular(gx, gy, stride):
            return brute_volume(self.grids[b], lut, gx[0, 0] + gy[0, 0] * ws, ws, ds, gx.shape[1], gx.shape[0], stride)
        return volume_at(self.grids[b], lut, (gx + gy * ws).ravel(), ds).reshape(gx.shape[0], gx.shape[1], lut.shape[0])

    def origins(self, b, search):
        """window origins base00 + lut[k, i] (int64, INVALID_SCAN readings dropped per angle) of a regular lattice"""
        gx, gy = self.cells(b, search)
        base00 = int(gx[0, 0] + gy[0, 0] * self.g.width_step)
        lut = self.lut(b, search)
        return [base00 + lut[k][lut[k] != INVALID_SCAN].astype(np.int64) for k in range(lut.shape[0])]


def random_scans(rng, B, laser_s, r_lo, r_hi, dropout=0.0):
    n = laser_s.n_readings
    ranges = rng.uniform(r_lo, r_hi, size=(B, n))
    if dropout:
        m = rng.random((B, n)) < dropout
        ranges[m] = np.where(rng.random(m.sum()) < 0.5, np.nan, np.inf)
    poses = np.column_stack([rng.uniform(-2, 2, B), rng.uniform(-2, 2, B), rng.uniform(-math.pi, math.pi, B)])
    return ranges, poses


def window_search(batch, side=None, stride=1, angle_offset=2 * D, angle_res=1 * D, pen=1, fine=0):
    """a Search around the centre of `side` x `side` grid cells (the handle's search window by default) on a stride-1
    or stride-2 lattice"""
    r = batch.resolution
    side = batch.g.search_side if side is None else side
    half = 0.5 * (side - 1) * r
    return abi.Search(half, half, stride * r, stride * r, angle_offset, angle_res, pen, fine)


# geometry: (search_size, resolution, smear, range_threshold)
SMALL = (1.5, 0.05, 0.03, 9.25)            # the benchmark's: 408 x 405 bytes, the whole grid in shared memory
BANDED = [(1.5, 0.05, 0.03, 12.0),          # the banded geometries of test_banded_window_kernel_large_grids
          (1.5, 0.025, 0.03, 9.25)]
PROBE_GEOMS = [SMALL] + BANDED


def probe_batch(geom, stride, seed, B=64):
    """B matches whose grids hold a few isolated non-zero cells: at window corners and one cell outside them (on both
    sides of 4x4-block edges, at every byte alignment of the origin), in the padding columns, at flat index 0 and
    data_size - 1, at both ends of rows (wrap), and one match with a cell in every row (every band seam and halo row of
    a banded sweep).  Readings reach beyond the grid so that windows leave it on every side."""
    search_size, res, smear, rt = geom
    params = abi.matcher_params(search_size, res, smear, rt)
    laser_s = make_laser(1081, rt=rt)
    rng = np.random.default_rng(seed)
    ranges, poses = random_scans(rng, B, laser_s, 0.3, rt * 1.6, dropout=0.03)
    bt = Batch(params, laser_s, ranges, poses)
    g = bt.g
    ws, ds, h = g.width_step, g.data_size, g.height
    se = window_search(bt, stride=stride)
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    fx, fy = stride * (nx - 1) + 1, stride * (ny - 1) + 1  # footprint of a window in cells
    for b in range(B):
        grid = bt.grids[b]
        val = lambda: int(rng.integers(1, 101))  # noqa: E731
        mode = b % 8
        if mode == 0:
            grid[0], grid[ds - 1] = val(), val()
        elif mode == 1:  # padding columns x in [width, width_step)
            for _ in range(3):
                grid[int(rng.integers(0, h)) * ws + int(rng.integers(g.width, ws))] = val()
        elif mode == 2:  # last byte of a row and first byte of the next
            for _ in range(2):
                y = int(rng.integers(0, h - 1))
                grid[y * ws + ws - 1], grid[(y + 1) * ws] = val(), val()
        elif mode == 3:  # a cell in every row: band seams and halo rows
            cols = rng.integers(0, ws, size=h)
            grid[np.arange(h) * ws + cols] = rng.integers(1, 101, size=h)
        else:
            # window-corner probes: beams whose window lies inside the grid without wrapping, with its last column
            # (mode 4) / last row (mode 5) starting a 4x4 block, or any (modes 6, 7); one cell at a corner or one cell
            # past an edge of that window
            origins = bt.origins(b, se)
            k = int(rng.integers(0, len(origins)))
            a = origins[k]
            y, x = np.floor_divide(a, ws), np.mod(a, ws)
            ok = (a >= 0) & (x + fx <= ws) & (y + fy <= h)
            if mode == 4:
                ok &= (x + fx - 1) % 4 == 0
            elif mode == 5:
                ok &= (y + fy - 1) % 4 == 0
            cand = a[ok]
            spots = [(0, 0), (0, fx - 1), (fy - 1, 0), (fy - 1, fx - 1), (-1, 0), (0, -1), (fy, fx - 1), (fy - 1, fx)]
            for a0 in rng.choice(cand, size=min(4, len(cand)), replace=False):
                r, c = spots[int(rng.integers(0, 4 if mode in (4, 5) else len(spots)))]
                p = int(a0) + r * ws + c
                if 0 <= p < ds:
                    grid[p] = val()
    return bt, se


def uniform_batch(n, value, B=2, seed=5, rt=4.0):
    """B matches of n beams on a grid that holds `value` in every byte, readings inside the grid: every window is an
    interior one and no window is empty."""
    params = abi.matcher_params(1.5, 0.05, 0.03, rt)
    laser_s = make_laser(n, rt=rt)
    rng = np.random.default_rng(seed + n)
    ranges, poses = random_scans(rng, B, laser_s, 0.5, rt - 0.8)
    bt = Batch(params, laser_s, ranges, poses)
    bt.grids[:] = value
    return bt, window_search(bt, angle_offset=1 * D, angle_res=1 * D)


def class_sizes(bt, b, search):
    """beams per (angle, byte alignment a & 3) of match b: the window kernel's classes when every window is interior"""
    return np.array([np.bincount(a & 3, minlength=4) for a in bt.origins(b, search)])


def degenerate_smear_inputs(sigma_cells, seed=11, n_base=4, B=3):
    """MatchScan inputs whose smear deviation is sigma_cells x resolution, with n_base overlapping base scans and
    NaN / inf dropouts"""
    res = 0.05
    laser_s = synth.Laser(range_threshold=4.0)
    params = abi.matcher_params(1.5, res, sigma_cells * res, 4.0)
    world, poses, ranges = synth.make_trajectory(seed, n_base + B, laser_s, step_xy=0.08, step_th_deg=3)
    rng = np.random.default_rng(seed)
    ranges = ranges.copy()
    drop = rng.random(ranges.shape) < 0.03
    ranges[drop] = np.where(rng.random(drop.sum()) < 0.5, np.nan, np.inf)
    cur_r, cur_p = ranges[n_base:], poses[n_base:] + rng.uniform(-0.04, 0.04, size=(B, 3))
    return params, laser_s, cur_r, cur_p, np.stack([ranges[:n_base]] * B), np.stack([poses[:n_base]] * B)


def rounding_tie_center(bt, b, search):
    """A search centre of match b whose candidate lattice is irregular: (cx + x - gox) * scale lands on .5 for some
    candidates and rounds the other way for others.  Tried on half-cell positions and their neighbouring doubles."""
    stride = search_stride(search, bt.resolution)
    gox, goy = bt.offs[b]
    for j in range(0, 40):
        for dx in (0, 1, -1, 2, -2):
            cx = gox + (bt.g.roi_w // 2 + j + 0.5) * bt.resolution
            for _ in range(abs(dx)):
                cx = np.nextafter(cx, np.inf if dx > 0 else -np.inf)
            c = np.array([cx, goy + (bt.g.roi_h // 2 - j + 0.5) * bt.resolution, bt.centers[b][2]])
            if not is_regular(*lattice(c, bt.offs[b], search, bt.g, bt.resolution), stride):
                return c
    return None


def irregular_batch(stride, seed=21, B=6):
    """match 0: a rounding-tie centre (irregular lattice, generic sweep); match 1: a centre 50 m away (out of range);
    the others regular.  Dense random grids, so that any candidate summed at the wrong cell shows."""
    params = abi.matcher_params(*SMALL)
    laser_s = make_laser(1081)
    rng = np.random.default_rng(seed)
    ranges, poses = random_scans(rng, B, laser_s, 0.3, 9.0, dropout=0.02)
    bt = Batch(params, laser_s, ranges, poses)
    bt.grids[:] = rng.integers(0, 101, size=bt.grids.shape)
    se = window_search(bt, stride=stride)
    bt.centers[0] = rounding_tie_center(bt, 0, se)
    bt.centers[1, 0] += 50.0
    return bt, se


# (nx, ny, nA): every candidate ties on a uniform grid without penalty
TIE_SHAPES = [(1, 1, 511), (7, 1, 73), (1, 1, 512), (8, 8, 8), (2, 2, 128), (1, 1, 513), (3, 3, 57)]


def tie_batch(nx, ny, na, seed=31):
    params = abi.matcher_params(1.5, 0.05, 0.03, 4.0)
    laser_s = make_laser(360, rt=4.0)
    rng = np.random.default_rng(seed)
    ranges, poses = random_scans(rng, 2, laser_s, 0.5, 2.5)
    poses[:, :2] += np.array([[1.2345678901, -2.3456789012], [0.1234567, 3.3333333]])
    bt = Batch(params, laser_s, ranges, poses)
    bt.grids[:] = GRID_OCCUPIED
    r = bt.resolution
    ar = 0.05 * D
    se = abi.Search(0.5 * (nx - 1) * r, 0.5 * (ny - 1) * r, r, r, 0.5 * (na - 1) * ar, ar, 0, 0)
    return bt, se


def tie_sums(bt, b, search):
    """the tied poses' x / y sums of the reference order (y, x, theta), and as k_reduce's fixed-order tree forms them
    beyond RED_MAX_TIES ties: thread t sums cells t, t + 512, ... over theta, then a pairwise tree over the threads"""
    nx, ny, na = (abi.n_steps(search.offset_x, search.res_x), abi.n_steps(search.offset_y, search.res_y),
                  abi.n_steps(search.angle_offset, search.angle_res))
    cx, cy = bt.centers[b][:2]
    xs = [cx + (-search.offset_x + ix * search.res_x) for ix in range(nx)]
    ys = [cy + (-search.offset_y + iy * search.res_y) for iy in range(ny)]
    seq = [0.0, 0.0]
    part = np.zeros((2, RED_THREADS))
    for c in range(nx * ny):
        iy, ix = divmod(c, nx)
        for _ in range(na):
            seq[0] += xs[ix]
            seq[1] += ys[iy]
            part[0, c % RED_THREADS] += xs[ix]
            part[1, c % RED_THREADS] += ys[iy]
    d = RED_THREADS // 2
    while d:
        part[:, :d] += part[:, d:2 * d]
        d //= 2
    return np.array(seq), part[:, 0].copy()


def tolerance_batch(seed=41):
    """n = 10 000 beams, all but 1-3 NaN: one unit of an integer sum is exactly 1e-6 of response, the DoubleEqual
    tolerance of the tie test and of the penalty's zero test.  Grids of 0 / 1 / 2 bytes give best sums of 1 and 2 with
    neighbours one unit below."""
    n = 10_000
    params = abi.matcher_params(1.5, 0.05, 0.03, 4.0)
    laser_s = make_laser(n, rt=4.0)
    rng = np.random.default_rng(seed)
    B = 6
    ranges = np.full((B, n), np.nan)
    poses = np.column_stack([rng.uniform(-1, 1, B), rng.uniform(-1, 1, B), rng.uniform(-3, 3, B)])
    for b in range(B):
        k = 1 + b % 3
        ranges[b, rng.choice(n, size=k, replace=False)] = rng.uniform(0.5, 3.0, size=k)
    bt = Batch(params, laser_s, ranges, poses)
    for b in range(B):
        m = rng.random(bt.g.data_size) < 0.25
        bt.grids[b][m] = 1 if b < 3 else rng.integers(1, 3, size=m.sum())
    return bt, window_search(bt, side=7, angle_offset=5 * D, angle_res=1 * D)


# ------------------------------------------------------------------------------------------------ CPU tests

def assert_references_agree(bt, search, matches):
    for b in matches:
        rc, res, sums = bt.oracle(b, search)
        assert rc == 0, (b, rc)
        assert np.array_equal(bt.brute(b, search), sums), b


@pytest.mark.parametrize("geom", PROBE_GEOMS, ids=["small", "banded-12m", "banded-0.025"])
@pytest.mark.parametrize("stride", [1, 2])
def test_probe_grids_premise(geom, stride):
    bt, se = probe_batch(geom, stride, seed=100 + stride)
    g = bt.g
    assert_references_agree(bt, se, range(0, bt.B, 7 if geom != SMALL else 3))
    if geom != SMALL:
        assert g.data_size > SMEM_OPTIN  # swept in row bands
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    ws = g.width_step
    # the special cells are inside windows of their match: flat index 0 / data_size - 1, padding columns, row wrap
    for b in (0, 1, 2, 8, 9, 10):
        origins = np.concatenate(bt.origins(b, se))
        nz = np.flatnonzero(bt.grids[b])
        assert any(covers(origins, p, ws, nx, ny, stride).any() for p in nz), b
    # window-corner probes at a block edge: some window's only non-zero cells lie in its last column, which starts a
    # 4x4 block, so a summed-area test one cell short would drop that window
    fx, fy = stride * (nx - 1) + 1, stride * (ny - 1) + 1
    hit = 0
    for b in range(4, bt.B, 8):
        nz = np.flatnonzero(bt.grids[b])
        py, px = nz // ws, nz % ws
        for a in np.concatenate(bt.origins(b, se)):
            y, x = divmod(int(a), ws)
            if a < 0 or x + fx > ws or (x + fx - 1) % 4:
                continue
            foot = (py >= y) & (py < y + fy) & (px >= x) & (px < x + fx)
            if foot.any() and (px[foot] == x + fx - 1).all() and any(covers(np.array([a]), p, ws, nx, ny, stride)[0]
                                                                     for p in nz[foot]):
                hit += 1
    assert hit > 0


@pytest.mark.parametrize("n", [2048, 4000, LIST_MAX_BEAMS])
def test_saturation_premise(n):
    bt, se = uniform_batch(n, 127)
    assert_references_agree(bt, se, [0])
    sizes = class_sizes(bt, 0, se)
    assert sizes.sum(axis=1).max() == n  # every reading valid and interior
    if n >= 4000:
        # more than 512 beams of one class: the accumulators flush mid-class, and without that flush 127 * 517 > 65535
        assert sizes.max() > WIN_FLUSH_BEAMS and sizes.max() * 127 > 65535
    assert n * 26 + 64 <= 200 * 1024 < (LIST_MAX_BEAMS + 1) * 26 + 64


@pytest.mark.parametrize("sigma", [10.0, 9.99, 9.98])
def test_degenerate_smear_premise(sigma):
    params, laser_s, cur_r, cur_p, bran, bpos = degenerate_smear_inputs(sigma)
    pm = port.PortMatcher(params, abi.laser_from(laser_s))
    K = pm.kernel()
    h = K.shape[0] // 2
    off_centre = np.delete(K.ravel(), h * K.shape[0] + h)
    assert (off_centre.max() == GRID_OCCUPIED) == (sigma >= 9.99), off_centre.max()
    assert np.isnan(bran).any() and np.isinf(bran).any()


@pytest.mark.parametrize("stride", [1, 2])
def test_irregular_lattice_premise(stride):
    bt, se = irregular_batch(stride)
    assert bt.centers[0] is not None
    for b in range(bt.B):
        gx, gy = bt.cells(b, se)
        inside = ((gx >= 0) & (gx < bt.g.width) & (gy >= 0) & (gy < bt.g.height)).all()
        assert inside == (b != 1), b
        if b != 1:
            assert is_regular(gx, gy, stride) == (b != 0), b
    rc, _, _ = bt.oracle(1, se)
    assert rc == abi.B2S_ERR_OUT_OF_RANGE
    assert_references_agree(bt, se, [0, 2])


@pytest.mark.parametrize("shape", TIE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_tie_count_premise(shape):
    nx, ny, na = shape
    bt, se = tie_batch(nx, ny, na)
    assert (abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y),
            abi.n_steps(se.angle_offset, se.angle_res)) == shape
    rc, res, sums = bt.oracle(0, se)
    assert rc == 0 and res.tie_count == nx * ny * na
    assert np.array_equal(bt.brute(0, se), sums)
    assert (sums == sums.flat[0]).all()
    seq, tree = tie_sums(bt, 0, se)
    total = nx * ny * na
    assert np.array_equal(seq / total, np.array(res.pose[:2]))  # the restatement sums in reference order
    if total == RED_MAX_TIES and nx * ny > 1:
        # the tree order would give other bits: a test of bit-equality sees which of the two ran
        assert not np.array_equal(seq / total, tree / total)


def test_tolerance_premise():
    bt, se = tolerance_batch()
    n = bt.laser.n_readings
    assert 1.0 / (n * GRID_OCCUPIED) == 1e-6  # one unit of a sum is the DoubleEqual tolerance
    bests = set()
    for b in range(bt.B):
        rc, res, sums = bt.oracle(b, se)
        assert rc == 0
        assert np.array_equal(bt.brute(b, se), sums)
        best = int(sums.max())
        bests.add(best)
        assert (sums == best - 1).any(), b  # neighbours one unit (1e-6 of response) below the best
    assert {1, 2} <= bests


def test_beam_count_beyond_add_scan_shared_memory():
    """k_add_scan stages 25 bytes per beam: 12 000 beams do not fit in an H100's opt-in shared memory, so the handle
    must build those grids another way"""
    assert 25 * 12_000 + 20 > SMEM_OPTIN >= 25 * 9_000 + 20
