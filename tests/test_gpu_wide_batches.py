"""The batch-taking handles whose kernels put the batch on grid y, past gridDim.y's limit of 65 535: the Karto matcher
(k_grid_pool, k_sweep_generic), the batched Hector processor (k_hs_mark, k_hs_apply) and the batched occupancy-grid
build (k_occ_ros_grids).  Each kernel strides over the batch on y, so a grid row serves items b, b + 65 535, ...

Every handle is fed K = 23 distinct sources, row b taking source b mod 23.  Neither 65 535 nor 65 536 is a multiple of
23, so a row computed with another row's index (b mod 65 535, b - 65 536, a clamped b) carries another source's answer.
Each source's answer is made twice: on a small handle of the 23 sources and by an independent reference (the brute-force
volume and the C restatement, PortHectorProcessor, the brute-force ray trace).  Every row of a wide batch must equal its
source's small-handle answer bit for bit; the heavier per-row read-backs (volumes, maps) are checked on rows 0, 65 534,
65 535, 65 536, the last row and 200 seeded random rows.

Batch sizes: 65 535 (one row per item), 65 536 (the first past the limit) and, where it fits in about 4 GB of device
memory, more than 2 x 65 535 (rows that serve three items).  The tests without the gpu mark check on the CPU that the
sources still reach the edges they exist for.
"""
import numpy as np
import pytest

import hector_cases as hc
import karto_volume_reference as kv
import raytrace_cases as rc
import raytrace_reference as rr
import test_prune_bound as pb
from karto_volume_reference import D, abi
from oracle import port
from test_gpu_matcher_edges import check_batch

K = 23            # distinct sources; row b takes source b % K
GRID_Y = 65_535   # gridDim.y's limit
TOL = 1e-9
gpu = pytest.mark.gpu


def sources_of(B):
    return np.arange(B) % K


def sampled_rows(B, seed=7):
    """rows 0, 65 534, 65 535, 65 536 and the last (those that exist) and 200 seeded random rows"""
    fixed = [b for b in (0, GRID_Y - 1, GRID_Y, GRID_Y + 1, B - 1) if b < B]
    rnd = np.random.default_rng(seed).choice(B, size=min(200, B), replace=False)
    return sorted(set(fixed) | set(int(b) for b in rnd))


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.fixture(scope="module")
def M(pkg):
    m = pkg.load("matcher")
    assert m.device_count() > 0, "no CUDA device: the product path has no fallback"
    return m


# ------------------------------------------------------------------------------------------------ Karto matcher

MATCH_GEOM = (0.2, 0.05, 0.03, 0.6)   # search 0.2 m, 0.05 m cells, smear 0.03 m, range threshold 0.6 m: 33 x 33 grids
TIE, FAR = 21, 22                     # the rounding-tie centre (irregular lattice) and the centre 50 m away
# grids of the match's own scan, whose pruning depends on the pool: source 8 is row 65 535's (65 535 = 8 mod 23), the
# first row a second pass of the y loop serves
OWN_SCAN = (8, 16, 17, 18, 19)


def matcher_sources(seed=2024):
    """K matches of 32 beams: probe grids (isolated cells at both ends of the data, in the padding columns, at row
    ends, one in every row, at window corners), grids holding the match's own scan (what add_scans of the same scan
    makes: the sweep prunes every angle it does not probe), a grid of saturated plateaus (what a degenerate smear makes),
    a rounding-tie centre on a dense grid and a centre out of range.  The search has 33 angles, enough for the plan to
    prune (PRUNE_MIN_ANGLES = 32, karto_sweep_plan.cuh): selector 0 then bounds the angles from k_grid_pool's pools."""
    search_size, res, smear, rt = MATCH_GEOM
    params = abi.matcher_params(search_size, res, smear, rt)
    laser_s = kv.make_laser(32, rt=rt)
    rng = np.random.default_rng(seed)
    ranges, poses = kv.random_scans(rng, K, laser_s, 0.05, rt * 1.6, dropout=0.05)
    bt = kv.Batch(params, laser_s, ranges, poses)
    g = bt.g
    ws, ds, h = g.width_step, g.data_size, g.height
    se = kv.window_search(bt, angle_offset=16 * D, angle_res=1 * D)
    nx, ny = abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.offset_y, se.res_y)
    na = abi.n_steps(se.angle_offset, se.angle_res)
    val = lambda: int(rng.integers(1, 101))  # noqa: E731
    for b in range(K):
        grid = bt.grids[b]
        if b in OWN_SCAN:  # every valid reading's cell, seen from the centre candidate at the centre angle
            gx, gy = bt.cells(b, se)
            o = bt.lut(b, se)[na // 2]
            o = o[o != kv.INVALID_SCAN].astype(np.int64) + int(gx[ny // 2, nx // 2] + gy[ny // 2, nx // 2] * ws)
            grid[o[(o >= 0) & (o < ds)]] = kv.GRID_OCCUPIED
        elif b < 16:
            mode = b % 8
            if mode == 0:
                grid[0], grid[ds - 1] = val(), val()
            elif mode == 1:
                for _ in range(3):
                    grid[int(rng.integers(0, h)) * ws + int(rng.integers(g.width, ws))] = val()
            elif mode == 2:
                for _ in range(2):
                    y = int(rng.integers(0, h - 1))
                    grid[y * ws + ws - 1], grid[(y + 1) * ws] = val(), val()
            elif mode == 3:
                grid[np.arange(h) * ws + rng.integers(0, ws, size=h)] = rng.integers(1, 101, size=h)
            else:  # a window corner of some beam, or one cell past it
                a = np.concatenate(bt.origins(b, se))
                a = a[(a >= 0) & (a % ws + nx <= ws) & (a // ws + ny <= h)]
                spots = [(0, 0), (0, nx - 1), (ny - 1, 0), (ny - 1, nx - 1), (-1, 0), (0, -1), (ny, nx - 1), (ny - 1, nx)]
                for a0 in rng.choice(a, size=min(4, len(a)), replace=False):
                    r, c = spots[int(rng.integers(0, len(spots)))]
                    if 0 <= int(a0) + r * ws + c < ds:
                        grid[int(a0) + r * ws + c] = val()
        elif b == 20:  # plateaus of GRID_OCCUPIED
            for _ in range(6):
                y, x = int(rng.integers(0, h - 4)), int(rng.integers(0, ws - 4))
                for r in range(4):
                    grid[(y + r) * ws + x:(y + r) * ws + x + 4] = kv.GRID_OCCUPIED
        else:
            grid[:] = rng.integers(0, 101, size=ds) * (rng.random(ds) < 0.4)
    bt.centers[TIE] = kv.rounding_tie_center(bt, TIE, se)
    bt.centers[FAR, 0] += 50.0
    return bt, se


def pruned_angles(bt, se):
    """[K] angles the pruned sweep leaves out of each match, by the numpy restatement of the bound and the selection
    rule (test_prune_bound.py) on the restatement's volume; 0 for the out-of-range and the irregular match, which are
    not pruned"""
    na = abi.n_steps(se.angle_offset, se.angle_res)
    out = np.zeros(K, np.int64)
    for b in range(K):
        if b in (TIE, FAR):
            continue
        rc_, _, sums = bt.oracle(b, se)
        gx, gy = bt.cells(b, se)
        base00 = int(gx[0, 0] + gy[0, 0] * bt.g.width_step)
        frac = pb.check_case(bt.grids[b], bt.g, bt.lut(b, se), base00, sums, bt.laser.n_readings, se, bt.params,
                             bt.centers[b][2])
        out[b] = round(frac * na)
    return out


def pruned_count(m, B, na):
    """angles the last correlate_scan left out, summed over its matches"""
    return round(m.last_pruned_frac() * B * na)


def matcher_handle(M, bt, B, idx):
    m = M.ScanMatcher(bt.params, bt.laser, max_batch=B, max_base_scans=1)
    m.set_scans(bt.ranges[idx], bt.poses[idx])
    m.set_grids(bt.grids[idx], bt.offs[idx])
    return m


KERNELS = (0, 3, 1)  # auto (pruned: angles bounded from k_grid_pool's pooled grids), dense window, generic


@pytest.fixture(scope="module")
def matcher_small(M):
    """each source's volumes and results on a handle of the K sources, checked against both references"""
    bt, se = matcher_sources()
    dims = (abi.n_steps(se.offset_y, se.res_y), abi.n_steps(se.offset_x, se.res_x), abi.n_steps(se.angle_offset, se.angle_res))
    m = matcher_handle(M, bt, K, np.arange(K))
    pruned = pruned_angles(bt, se)
    out = {}
    for kernel in KERNELS:
        m.set_kernel(kernel)
        res = check_batch(m, bt, se)
        vols = [m.response_sums(b, dims) if res[3][b] == 0 else None for b in range(K)]
        out[kernel] = (res, vols, m.last_timing()["path"])
        assert pruned_count(m, K, dims[2]) == (pruned.sum() if kernel == 0 else 0), kernel
    # the pruned sweep's results are the dense sweep's, byte for byte
    assert all(a.tobytes() == d.tobytes() for a, d in zip(out[0][0], out[3][0]))
    m.close()
    return bt, se, dims, out, pruned


def test_matcher_sources_premise():
    """the tie centre's lattice is irregular, the far centre out of range, every other lattice regular and in range;
    the brute-force volume equals the restatement's on every in-range source; the sources differ"""
    bt, se = matcher_sources()
    for b in range(K):
        gx, gy = bt.cells(b, se)
        inside = ((gx >= 0) & (gx < bt.g.width) & (gy >= 0) & (gy < bt.g.height)).all()
        assert inside == (b != FAR), b
        if b != FAR:
            assert kv.is_regular(gx, gy, 1) == (b != TIE), b
    assert bt.oracle(FAR, se)[0] == abi.B2S_ERR_OUT_OF_RANGE
    kv.assert_references_agree(bt, se, [b for b in range(K) if b != FAR])
    nonzero = [b for b in range(K) if b != FAR and bt.brute(b, se).any()]
    assert len(nonzero) >= 15, nonzero
    assert len({bt.grids[b].tobytes() for b in range(K)}) == K
    assert GRID_Y % K and (GRID_Y + 1) % K and (2 * GRID_Y + 1) % K
    pruned = pruned_angles(bt, se)
    na = abi.n_steps(se.angle_offset, se.angle_res)
    assert na >= 32 and (pruned[list(OWN_SCAN)] == na - pb.PROBE).all(), pruned
    assert GRID_Y % K == OWN_SCAN[0]


@gpu
@pytest.mark.parametrize("B", [GRID_Y, GRID_Y + 1, 2 * GRID_Y + 1])
def test_matcher_correlate_wide(M, matcher_small, B):
    """correlate_scan on every kernel path: every row's status, tie count, response, pose and covariance equal its
    source's on the small handle bit for bit, and the sampled rows' integer volumes equal the brute-force volume.  On
    selector 0 angles are pruned on bounds read from every row's pooled grid (k_grid_pool): the angles left out add up
    to its source's count over every row, so a row whose pool were missing or another row's would show in that sum
    if not in its results."""
    bt, se, dims, small, pruned = matcher_small
    idx = sources_of(B)
    m = matcher_handle(M, bt, B, idx)
    ok = small[0][0][3][idx] == 0
    for kernel in KERNELS:
        m.set_kernel(kernel)
        resp, pose, cov, status, ties = m.correlate_scan(bt.centers[idx], se)
        (s_resp, s_pose, s_cov, s_status, s_ties), vols, path = small[kernel]
        assert m.last_timing()["path"] == path, kernel
        assert pruned_count(m, B, dims[2]) == (pruned[idx].sum() if kernel == 0 else 0), kernel
        assert np.array_equal(status, s_status[idx]), (kernel, np.flatnonzero(status != s_status[idx])[:8])
        assert np.array_equal(ties, s_ties[idx]), (kernel, np.flatnonzero(ties != s_ties[idx])[:8])
        for got, want in ((resp, s_resp), (pose, s_pose), (cov, s_cov)):
            assert bits_equal(got[ok], want[idx][ok]), kernel
        for b in sampled_rows(B):
            if status[b] == 0:
                vol = m.response_sums(b, dims)
                assert np.array_equal(vol, vols[idx[b]]), (kernel, b)
                assert np.array_equal(vol, bt.brute(idx[b], se)), (kernel, b)
    assert (status[idx == FAR] == abi.B2S_ERR_OUT_OF_RANGE).all()
    m.close()


def match_sources(seed=77):
    """K MatchScan inputs of 32 beams with two base scans each, near the current pose"""
    search_size, res, smear, rt = MATCH_GEOM
    params = abi.matcher_params(search_size, res, smear, rt)
    laser_s = kv.make_laser(32, rt=rt)
    rng = np.random.default_rng(seed)
    cur_r, cur_p = kv.random_scans(rng, K, laser_s, 0.1, 0.58, dropout=0.05)
    bran = np.clip(cur_r[:, None, :] + rng.uniform(-0.03, 0.03, size=(K, 2, 32)), 0.05, None)
    bpos = cur_p[:, None, :] + rng.uniform(-0.04, 0.04, size=(K, 2, 3))
    return params, abi.laser_from(laser_s), cur_r, cur_p, bran, bpos


@gpu
def test_matcher_match_scan_wide(M):
    """MatchScan (coarse, response expansion, fine stage with its angular covariance) on 131 071 matches whose grids
    the handle builds from base scans: every row equals its source on a handle of the K sources bit for bit, which
    equals the restatement's MatchScan; the sampled rows' grids equal the source's"""
    params, laser, cur_r, cur_p, bran, bpos = match_sources()
    small = M.ScanMatcher(params, laser, max_batch=K, max_base_scans=2)
    s_res = small.match_scan_host(cur_r, cur_p, bran, bpos, True, True)
    s_grids = [small.grid(b) for b in range(K)]
    for b in range(K):
        pm = port.PortMatcher(params, laser)
        rc_, res = pm.match_scan(cur_r[b], cur_p[b], bran[b], bpos[b], True, True)
        assert s_res[3][b] == rc_ == 0, b
        assert np.array_equal(s_grids[b][0], pm.grid) and np.array_equal(s_grids[b][1], pm.grid_off), b
        assert abs(s_res[0][b] - res.response) <= TOL, b
        assert np.allclose(s_res[1][b], res.pose[:], rtol=0, atol=TOL), b
        assert np.allclose(s_res[2][b].ravel(), res.cov[:], rtol=0, atol=TOL), b
    assert (s_res[0] > 0).sum() >= K - 2
    small.close()
    B = 2 * GRID_Y + 1
    idx = sources_of(B)
    m = M.ScanMatcher(params, laser, max_batch=B, max_base_scans=2)
    res = m.match_scan_host(cur_r[idx], cur_p[idx], bran[idx], bpos[idx], True, True)
    for got, want in zip(res, s_res):
        assert bits_equal(got, want[idx])
    for b in sampled_rows(B):
        grid, off = m.grid(b)
        assert np.array_equal(grid, s_grids[idx[b]][0]) and np.array_equal(off, s_grids[idx[b]][1]), b
    m.close()


# ------------------------------------------------------------------------------------------------ Hector batch

HECTOR_KW = dict(size_x=32, size_y=32, resolution=0.1, start=(0.5, 0.5), levels=2, **hc.GATE)
HECTOR_CAP = 64
STEPS = 3
STILL, EMPTY_STEP, FULL = 0, 1, 2   # a source that does not move (its gate stays shut), one with an empty scan, one at the cap


def hector_sources(seed=404):
    """K self-driven streams of three scans: a rectangular room of 20-64 wall points (level-0 cells, laser frame) seen
    from a robot that moves 0.15-0.3 m and turns a little between scans (the gate opens), except source STILL, which
    sees the same scan three times (the gate stays shut after the first), and source EMPTY_STEP, whose second scan has
    no points.  Returns ([scans [STEPS][n, 2]], first poses [K, 3])."""
    rng = np.random.default_rng(seed)
    streams, firsts = [], []
    for s in range(K):
        hw, hh = rng.uniform(7.0, 11.0, size=2)  # half sizes of the room in cells: the robot stays well inside 32 x 32
        n = HECTOR_CAP if s == FULL else int(rng.integers(20, HECTOR_CAP + 1))
        t = rng.uniform(0.0, 1.0, size=n)
        side = rng.integers(0, 4, size=n)
        wall = np.stack([np.where(side < 2, np.where(side == 0, -hw, hw), (2 * t - 1) * hw),
                         np.where(side < 2, (2 * t - 1) * hh, np.where(side == 2, -hh, hh))], 1)
        pose = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(-0.4, 0.4)])
        firsts.append(pose.astype(np.float32))
        scans = []
        for i in range(STEPS):
            if i and s != STILL:
                step = rng.uniform(0.15, 0.3)
                d = rng.uniform(-np.pi, np.pi)
                pose = pose + np.array([step * np.cos(d), step * np.sin(d), rng.uniform(-0.05, 0.05)])
            c, sn = np.cos(pose[2]), np.sin(pose[2])
            rel = wall - pose[:2] / HECTOR_KW["resolution"]  # world cells relative to the robot
            pts = np.stack([c * rel[:, 0] + sn * rel[:, 1], -sn * rel[:, 0] + c * rel[:, 1]], 1).astype(np.float32)
            scans.append(np.zeros((0, 2), np.float32) if (s == EMPTY_STEP and i == 1) else pts)
        streams.append(scans)
    return streams, np.stack(firsts)


def hector_reference(streams, firsts):
    """the restatement over each source alone: processors, poses [K, STEPS, 3], covariances [K, STEPS, 3, 3], gate
    decisions [K, STEPS]"""
    procs, poses, covs, flags = [], [], [], []
    for s in range(K):
        c = port.PortHectorProcessor(**HECTOR_KW)
        est, ps, cs, fs = firsts[s], [], [], []
        for i in range(STEPS):
            est, cov = c.update(streams[s][i], (0, 0), est)
            ps.append(np.asarray(est, np.float32)), cs.append(np.asarray(cov, np.float32).reshape(3, 3))
            fs.append(c.map_updated)
        procs.append(c), poses.append(ps), covs.append(cs), flags.append(fs)
    return procs, np.array(poses, np.float32), np.array(covs, np.float32), np.array(flags, bool)


def test_hector_sources_premise():
    """every source updates its map on the first scan; STILL's gate stays shut afterwards, the moving sources' opens"""
    streams, firsts = hector_sources()
    procs, poses, covs, flags = hector_reference(streams, firsts)
    assert flags[:, 0].all()
    assert not flags[STILL, 1:].any()
    # a shut gate shows as a last map-update pose other than the last scan-match pose (update_batch_device returns no flags)
    assert not hc.same_bits(poses[STILL, 1], poses[STILL, 0])
    assert flags[[s for s in range(K) if s not in (STILL, EMPTY_STEP)], 1:].sum() >= 2 * (K - 2) - 4
    assert len(streams[FULL][0]) == HECTOR_CAP and len(streams[EMPTY_STEP][1]) == 0
    assert np.isfinite(poses).all()
    for c in procs:
        c.close()


@pytest.fixture(scope="module")
def H(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector")


def step_batch(g, scans, hints):
    """update_batch over the steps; -> per step (poses [B, 3], covs [B, 3, 3], flags [B])"""
    return [g.update_batch(scans[i], (0, 0), hints if i == 0 else None) for i in range(STEPS)]


@pytest.fixture(scope="module")
def hector_small(H):
    """the K sources on one handle, checked against the restatement bit for bit; its results and maps"""
    streams, firsts = hector_sources()
    procs, poses, covs, flags = hector_reference(streams, firsts)
    g = H.HectorSlam(batch=K, max_points=HECTOR_CAP, **HECTOR_KW)
    steps = step_batch(g, [[streams[s][i] for s in range(K)] for i in range(STEPS)], firsts)
    last, levels = [], []
    for s in range(K):
        for i, (p, c, u) in enumerate(steps):
            assert hc.same_bits(p[s], poses[s, i]) and u[s] == flags[s, i], (s, i)
            assert hc.same_bits(c[s], covs[s, i]), (s, i)
        a, u = g.last_poses(s)
        upd = np.flatnonzero(flags[s])
        assert hc.same_bits(a, poses[s, -1]) and hc.same_bits(u, poses[s, upd[-1]]), s
        last.append((a, u))
        levels.append([g.level_of(s, lvl) for lvl in range(HECTOR_KW["levels"])])
        for lvl in range(HECTOR_KW["levels"]):
            assert hc.cell_mismatch(levels[s][lvl], procs[s].level(lvl))[0] == 0, (s, lvl)
        procs[s].close()
    g.close()
    return streams, firsts, steps, last, levels


def check_last_poses(g, B, last, what):
    """every row's last scan-match and last map-update pose equal its source's, last [K] of (match, update) poses"""
    idx = sources_of(B)
    for b in range(B):
        a, u = g.last_poses(b)
        assert hc.same_bits(a, last[idx[b]][0]) and hc.same_bits(u, last[idx[b]][1]), (what, b)


def check_hector_rows(g, B, last, levels, what):
    check_last_poses(g, B, last, what)
    idx = sources_of(B)
    for b in sampled_rows(B):
        for lvl in range(HECTOR_KW["levels"]):
            assert hc.cell_mismatch(g.level_of(b, lvl), levels[idx[b]][lvl])[0] == 0, (what, b, lvl)


@gpu
@pytest.mark.parametrize("B", [GRID_Y, GRID_Y + 2])
def test_hector_update_batch_wide(H, hector_small, B):
    """three update_batch steps: every row's poses, covariances and gate decisions after each step and its last poses
    equal its source's on the small handle bit for bit, and the sampled rows' maps on both levels too"""
    streams, firsts, steps, last, levels = hector_small
    idx = sources_of(B)
    g = H.HectorSlam(batch=B, max_points=HECTOR_CAP, **HECTOR_KW)
    got = step_batch(g, [[streams[s][i] for s in idx] for i in range(STEPS)], firsts[idx])
    for i in range(STEPS):
        for x, y in zip(got[i], steps[i]):
            assert bits_equal(x, y[idx]), (i, np.flatnonzero((x != y[idx]).reshape(B, -1).any(1))[:8])
    assert not got[1][2][idx == STILL].any() and got[1][2][idx != STILL].any()
    check_hector_rows(g, B, last, levels, "update_batch")
    g.close()


@gpu
def test_hector_update_batch_device_and_stream_wide(H, hector_small):
    """the same three steps through update_batch_device (torch tensors on the device) and through one
    process_stream_batch call, on 65 537 processors.  update_batch_device returns nothing to the host, so after each of
    its steps every row's pose is read back as its last scan-match pose and its gate decision as its last map-update
    pose (this step's pose if the gate opened, the earlier one if not), both equal to its source's step on the small
    handle; the covariances of those steps are not read back by any entry point and are checked through update_batch
    and process_stream_batch only."""
    import torch
    streams, firsts, steps, last, levels = hector_small
    B = GRID_Y + 2
    idx = sources_of(B)
    pts = np.zeros((K, STEPS, HECTOR_CAP, 2), np.float32)
    cnt = np.zeros((K, STEPS), np.int32)
    for s in range(K):
        for i in range(STEPS):
            pts[s, i, :len(streams[s][i])] = streams[s][i]
            cnt[s, i] = len(streams[s][i])
    g = H.HectorSlam(batch=B, max_points=HECTOR_CAP, **HECTOR_KW)
    d_pts = torch.as_tensor(np.ascontiguousarray(pts[idx].transpose(1, 0, 2, 3)), device="cuda")
    d_cnt = torch.as_tensor(np.ascontiguousarray(cnt[idx].T), device="cuda")
    d_hints = torch.as_tensor(firsts[idx], device="cuda")
    torch.cuda.synchronize()
    s_poses = np.stack([p for p, _, _ in steps], 1)  # [K, STEPS, 3]
    s_flags = np.stack([u for _, _, u in steps], 1)
    for i in range(STEPS):
        g.update_batch_device(d_pts[i].data_ptr(), d_cnt[i].data_ptr(), int(cnt[:, i].max()), (0, 0),
                              d_hints.data_ptr() if i == 0 else None)
        g.sync()
        upd = [np.flatnonzero(s_flags[s, :i + 1])[-1] for s in range(K)]  # the first step always updates
        check_last_poses(g, B, [(s_poses[s, i], s_poses[s, upd[s]]) for s in range(K)], ("update_batch_device", i))
    check_hector_rows(g, B, last, levels, "update_batch_device")
    g.close()
    del d_pts, d_cnt, d_hints

    g = H.HectorSlam(batch=B, max_points=HECTOR_CAP, **HECTOR_KW)
    res, covs = g.process_stream_batch([streams[s] for s in idx], (0, 0), first_hints=firsts[idx])
    for b in range(B):
        assert hc.same_bits(res[b][0], s_poses[idx[b]]) and np.array_equal(res[b][1], s_flags[idx[b]]), b
    assert hc.same_bits(covs, steps[-1][1][idx])
    check_hector_rows(g, B, last, levels, "process_stream_batch")
    g.close()


# ------------------------------------------------------------------------------------------------ occupancy grids

OCC_LASER = dict(n=8, min_angle=-np.pi, ares=2 * np.pi / 8, min_range=0.05, max_range=2.0, threshold=1.2)
OCC_RES = (0.1, 0.1, 0.2, 0.05)
ALL_INVALID = 4                      # a source whose readings are all invalid: a grid of width and height 0
# live grids -> rows left without scans (past 65 535); n_grids = live + len(zero rows)
OCC_CASES = {GRID_Y: (), GRID_Y + 1: (GRID_Y + 1, GRID_Y + 2),
             2 * GRID_Y + 18: (GRID_Y + 1, GRID_Y + 2, GRID_Y + 65, 100_001, 2 * GRID_Y + 21)}


def occ_sources(seed=99):
    """K grids of one or two 8-beam scans (float32 ranges, some past the range threshold or the maximum, some NaN or
    below the minimum) at 0.05-0.2 m"""
    rng = np.random.default_rng(seed)
    laser = rc.laser(**OCC_LASER)
    ranges, poses, res = [], [], []
    for s in range(K):
        n = 1 + s % 2
        r = rng.uniform(0.1, 2.2, size=(n, 8)).astype(np.float32)
        r[rng.random((n, 8)) < 0.1] = np.nan
        if s == ALL_INVALID:
            r[:] = np.nan
        ranges.append(r)
        poses.append(np.column_stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(-np.pi, np.pi, n)]))
        res.append(OCC_RES[s % len(OCC_RES)])
    return laser, ranges, poses, np.array(res)


def occ_rows(live):
    zero = OCC_CASES[live]
    G = live + len(zero)
    idx = sources_of(G)
    return G, idx, np.isin(np.arange(G), zero)


def test_occ_sources_premise():
    """the zero rows lie past 65 535 and keep the live count; the all-invalid source makes a 0 x 0 grid"""
    laser, ranges, poses, res = occ_sources()
    for live, zero in OCC_CASES.items():
        G, idx, empty = occ_rows(live)
        assert (~empty).sum() == live and all(GRID_Y < z < G for z in zero)
    assert max(OCC_CASES) > 2 * GRID_Y
    b = rr.occupancy_grid(laser, ranges[ALL_INVALID].astype(np.float64), poses[ALL_INVALID], res[ALL_INVALID])
    assert (b["width"], b["height"]) == (0, 0)
    known = 0
    for s in range(K):
        if s != ALL_INVALID:
            b = rr.occupancy_grid(laser, ranges[s].astype(np.float64), poses[s], res[s])
            assert b["width"] * b["height"] > 0, s
            known += int((b["cells"] != rr.UNKNOWN).any())
    assert known >= 5


@pytest.fixture(scope="module")
def O(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("occgrid")


@pytest.fixture(scope="module")
def occ_small(O):
    """the K grids in one batched build, checked against CreateFromScans per source and the brute-force ray trace"""
    laser, ranges, poses, res = occ_sources()
    out = O.create_from_scans_batch(laser, ranges, poses, res)
    for s in range(K):
        info, payload = out[s]
        r64 = ranges[s].astype(np.float64)
        one = O.OccupancyGrid(laser, r64, poses[s], res[s])
        a, b = one.arrays(), rr.occupancy_grid(laser, r64, poses[s], res[s])
        for ref in (a, b):
            assert (info["width"], info["height"], info["width_step"]) == (ref["width"], ref["height"], ref["width_step"]), s
            assert np.allclose(info["offset"], ref["offset"], rtol=0, atol=TOL) and info["cell_visits"] == ref["cell_visits"], s
        assert np.array_equal(info["offset"], a["offset"]), s
        want = rr.karto_ros_map(b["cells"], b["width"], b["height"])
        assert np.array_equal(payload, want), s
        if info["width"] * info["height"]:
            assert np.array_equal(payload, one.ros_map()), s
        one.close()
    return laser, ranges, poses, res, out


@gpu
@pytest.mark.parametrize("live", list(OCC_CASES))
def test_occ_grid_batch_wide(O, occ_small, live):
    """every grid's info and payload equal its source's in the small build, and grids without scans are None without
    moving their neighbours"""
    laser, ranges, poses, res, small = occ_small
    G, idx, empty = occ_rows(live)
    out = O.create_from_scans_batch(laser, [ranges[s][:0] if e else ranges[s] for s, e in zip(idx, empty)],
                                    [poses[s][:0] if e else poses[s] for s, e in zip(idx, empty)], res[idx])
    assert len(out) == G
    for g in range(G):
        if empty[g]:
            assert out[g] is None, g
            continue
        info, payload = out[g]
        s_info, s_payload = small[idx[g]]
        assert info.keys() == s_info.keys()
        for k in info:
            assert np.array_equal(info[k], s_info[k]), (g, k)
        assert bits_equal(payload, s_payload), g
