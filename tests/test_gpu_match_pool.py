"""The Karto Mapper's shared match pool (MatchPool, csrc/karto_mapper.cu) at its capacity edges, on the device.

a. A matcher's device scan pool across its growths (256, 512 rows) and chains padded by repeating their last scan,
   against host readings and the CPU restatement.
b. The standalone Mapper (b2s_mapper_create, its own pool) against the same Mapper with the restatement's MatchScan, on
   every workload of tests/match_pool_cases.py: batches past 8 / 16 / 32, chains at and past 32 and 64, 530 pool rows,
   a loop handle re-created while the sequential handle keeps its rows.
c. The node batch (b2s_karto_node_create_batch): groups of more than 256 matches split into launches, a node's batch
   split across two launches, and a loop handle re-created in the middle of a call; every node equals its own
   single-node handle bit for bit.
tests/test_match_pool_premises.py shows, without a GPU, that these workloads reach those edges."""
import ctypes as C

import numpy as np
import pytest

import karto_node_cases as kc
import karto_volume_reference as kv
import match_pool_cases as mc
from oracle import port
from test_gpu_karto_node_batch import assert_same_node
from test_match_pool_premises import node_trace, straddle_traces

pytestmark = pytest.mark.gpu
TOL = 1e-9
KN, MP, abi, synth = mc.KN, mc.MP, mc.abi, mc.synth
M = mc.PKG.load("matcher")


def assert_results_close(got, rc, res, b, who):
    resp, pose, cov, status, _ = got
    assert status[b] == rc == 0, who
    assert abs(resp[b] - res.response) <= TOL, who
    assert np.abs(pose[b] - np.array(res.pose[:])).max() <= TOL, who
    assert np.abs(cov[b].ravel() - np.array(res.cov[:])).max() <= TOL, who


# ------------------------------------------------------------------------------------------------ a. matcher pool

def test_scan_pool_rows_across_its_growths():
    """530 rows appended one by one, matches in between; then chains whose rows lie on both sides of each growth"""
    laser = synth.Laser()
    al = abi.laser_from(laser)
    params = abi.matcher_params(0.5, 0.05, 0.03, 9.25)
    _, poses, ranges = synth.make_trajectory(31, 530, laser, step_xy=0.05, step_th_deg=1)
    pool = M.ScanMatcher(params, al, max_batch=2, max_base_scans=6)
    host = M.ScanMatcher(params, al, max_batch=2, max_base_scans=6)
    rng = np.random.default_rng(31)

    def both(cur, chains):
        cp = poses[cur] + rng.uniform(-0.03, 0.03, (len(cur), 3))
        pool.set_scans(ranges[cur], cp)
        pool.add_scans_pool(chains, np.stack([poses[c] for c in chains]))
        got = pool.match_scan()
        host.set_scans(ranges[cur], cp)
        host.add_scans(np.stack([ranges[c] for c in chains]), np.stack([poses[c] for c in chains]))
        want = host.match_scan()
        for b in range(len(cur)):
            assert np.array_equal(pool.grid(b)[0], host.grid(b)[0]), (cur, b)
        for x, y in zip(got, want):
            assert np.array_equal(x, y), cur
        return cp, got

    for i in range(530):
        assert pool.pool_append(ranges[i]) == i
        if i in (3, 254, 255, 256, 300, 511, 512, 513) or i % 97 == 0 and i >= 3:
            both([i, i - 1], [[i - 1, i - 2, i - 3] * 2, [0, i, i - 2] * 2])
    chains = [[0, 255, 256, 511, 512, 529], [529, 512, 511, 256, 255, 0]]
    cur = [257, 510]
    cp, got = both(cur, chains)
    for b in range(2):
        pm = port.PortMatcher(params, al)
        rc, res = pm.match_scan(ranges[cur[b]], cp[b], ranges[chains[b]], poses[chains[b]], True, True)
        grid, off = pool.grid(b)
        assert np.array_equal(off, pm.grid_off) and np.array_equal(grid, pm.grid), b
        assert_results_close(got, rc, res, b, b)
    with pytest.raises(M.B2SError) as e:
        pool.set_scans(ranges[cur], cp)
        pool.add_scans_pool([[0, 530]] * 2, np.stack([poses[[0, 1]]] * 2))
    assert e.value.status == abi.B2S_ERR_OUT_OF_RANGE
    pool.close(), host.close()


@pytest.mark.parametrize("sigma", [0.6, 10.0], ids=["staged", "degenerate_smear"])
def test_chain_padded_by_its_last_scan(sigma):
    """a chain of 1 or 4 base scans padded to 40 entries by repeating its last one (as the pool pads a group to its
    longest chain): grid bytes and MatchScan results equal the restatement's on the chain as it is, on the staged
    AddScan kernel and on the sequential one an off-centre smear value of 100 makes order-dependent"""
    params, laser_s, cur_r, cur_p, bran, bpos = kv.degenerate_smear_inputs(sigma)
    al = abi.laser_from(laser_s)
    pm0 = port.PortMatcher(params, al)
    assert (np.delete(pm0.kernel().ravel(), pm0.kernel().size // 2).max() == kv.GRID_OCCUPIED) == (sigma == 10.0)
    B, nb = bran.shape[:2]
    lengths = [1, nb, 1][:B]
    pad = [list(range(n)) + [n - 1] * (40 - n) for n in lengths]
    pr = np.stack([bran[b][pad[b]] for b in range(B)])
    pp = np.stack([bpos[b][pad[b]] for b in range(B)])
    m = M.ScanMatcher(params, al, max_batch=B, max_base_scans=40)
    for b in range(B):
        for i in range(nb):
            m.pool_append(bran[b][i])
    for pen in (True, False):
        m.set_scans(cur_r, cur_p)
        m.add_scans(pr, pp)
        host = m.match_scan(pen, True)
        host_grids = [m.grid(b)[0] for b in range(B)]
        m.set_scans(cur_r, cur_p)
        m.add_scans_pool([[b * nb + i for i in pad[b]] for b in range(B)], pp)
        pooled = m.match_scan(pen, True)
        for x, y in zip(host, pooled):
            assert np.array_equal(x, y)
        for b in range(B):
            pm = port.PortMatcher(params, al)
            n = lengths[b]
            rc, res = pm.match_scan(cur_r[b], cur_p[b], bran[b][:n], bpos[b][:n], pen, True)
            grid, off = m.grid(b)
            assert np.array_equal(off, pm.grid_off) and np.array_equal(grid, pm.grid), (sigma, b)
            assert np.array_equal(host_grids[b], pm.grid), (sigma, b)
            assert_results_close(pooled, rc, res, b, (sigma, pen, b))
    m.close()


# ------------------------------------------------------------------------------------------------ b. standalone Mapper

@pytest.mark.parametrize("name", list(mc.WORKLOADS))
def test_standalone_mapper_equals_the_restatement(name):
    wl = mc.WORKLOADS[name]()
    r, rec, fr, cr = mc.recorded(wl)
    assert rec.events()  # the workload's pool events: tests/test_match_pool_premises.py pins which
    m = MP.Mapper(wl.params, wl.al)
    fm, cm = mc.run(m, wl)
    assert np.array_equal(fr, fm) and np.abs(cr - cm).max() <= TOL
    pr, pm = r.poses(), m.poses()
    assert pr.shape == pm.shape and np.abs(pr - pm).max() <= TOL
    (ir, dr, vr), (im, dm, vm) = r.edges(), m.edges()
    assert np.array_equal(ir, im), "graph edges differ"
    assert np.abs(dr - dm).max() <= TOL and np.abs(vr - vm).max() <= TOL
    assert r.stats() == m.stats()
    r.close(), m.close()


# ------------------------------------------------------------------------------------------------ c. node batch

GEOM = kc.CASES["loops_small_windows"].geometry()


def single_timing(node):
    out = np.zeros(8)
    assert node.L.b2s_karto_node_last_timing(node.h, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
    return dict(zip(("rounds", "match_launches", "matches"), out[:3].tolist()))


def snapshot(mapper, got):
    """a node's outputs with its Mapper's graph now"""
    return dict(got, edges=mapper.edges(), stats=mapper.stats(), poses_now=mapper.poses())


def singles_at(params, rows, lengths):
    """one single-node handle over the recording in parts ending at each of `lengths` -> {S: its outputs on the first
    S scans and its Mapper's graph after them} (a node's run is causal)"""
    prm, _ = KN.node_params(params)
    node = KN.KartoNode(prm, GEOM, mc.IDENT)
    out, acc, at = {}, None, 0
    for S in sorted(set(lengths)):
        part = node.process(*(x[at:S] for x in rows))
        if acc is None:
            acc = part
        else:
            acc = {k: (acc[k] + part[k] if k == "maps" else np.concatenate([acc[k], part[k]])) for k in acc}
        out[S] = snapshot(node.mapper, acc)
        at = S
    node.close()
    return out


def run_batch(params_list, rows_list):
    prms = [KN.node_params(p)[0] for p in params_list]
    fleet = KN.KartoNodeBatch(prms, GEOM, [mc.IDENT] * len(prms))
    got = fleet.process(*([r[k] for r in rows_list] for k in range(3)))
    got = [snapshot(fleet.mapper(b), g) for b, g in enumerate(got)]
    timing = fleet.last_timing()
    fleet.close()
    return got, timing


def test_node_batch_of_300_splits_its_groups():
    c = kc.CASES["loops_small_windows"]
    p = mc.node_params(kc, map_update_interval=1.0)
    rows = (c.ranges, c.stamps, c.odom)
    prm, _ = KN.node_params(p)
    node = KN.KartoNode(prm, GEOM, mc.IDENT)
    want = snapshot(node.mapper, node.process(*rows))
    one = single_timing(node)
    node.close()
    got, timing = run_batch([p] * 300, [rows] * 300)
    for b in range(300):
        assert_same_node(got[b], want, b)
    assert timing["matches"] == 300 * one["matches"] > 0
    assert timing["match_launches"] >= 2 * one["match_launches"]
    assert timing["rounds"] == one["rounds"]


def test_node_batch_straddles_the_256_boundary():
    rec = mc.node_recordings(kc)["laps"]
    nodes = mc.straddle_nodes(kc, len(rec[0]))
    sim = mc.simulate_batch(straddle_traces(), 20)
    assert sim["straddles"]
    got, timing = run_batch([p for p, _ in nodes], [tuple(x[:S] for x in rec) for _, S in nodes])
    assert (timing["match_launches"], timing["matches"]) == (sim["launches"], sim["matches"])
    singles = {}
    for t in (1, 2, 3):
        ns = [(p, S) for p, S in nodes if p["throttle_scans"] == t]
        singles[t] = singles_at(ns[0][0], rec, [S for _, S in ns])
    for b, (p, S) in enumerate(nodes):
        assert_same_node(got[b], singles[p["throttle_scans"]][S], b)


@pytest.mark.parametrize("chunked", [False, True], ids=["one_call", "chunked"])
def test_node_batch_loop_handle_recreated_mid_call(chunked):
    recs = mc.node_recordings(kc)
    names, extra = ["laps", "dense"], [{}, mc.DENSE]
    params = [mc.node_params(kc, map_update_interval=1.0, **e) for e in extra]
    rows = [recs[n] for n in names]
    sim = mc.simulate_batch([node_trace(n)[0] for n in names], 20)
    assert [(g[1], g[2]) for g in sim["regrowth"]] == [(1, [0])] and sim["later"] == [0]
    wants = [singles_at(p, r, [len(r[0])])[len(r[0])] for p, r in zip(params, rows)]
    if not chunked:
        got, timing = run_batch(params, rows)
        assert (timing["match_launches"], timing["matches"]) == (sim["launches"], sim["matches"])
        for b in range(2):
            assert_same_node(got[b], wants[b], names[b])
        return
    prms = [KN.node_params(p)[0] for p in params]
    fleet = KN.KartoNodeBatch(prms, GEOM, [mc.IDENT] * 2)
    cuts = [[0, 90, 200, 240, 300], [0, 150, 238, 245, 260]]
    parts = []
    for k in range(len(cuts[0]) - 1):
        parts.append(fleet.process(*([r[i][cuts[b][k]:cuts[b][k + 1]] for b, r in enumerate(rows)] for i in range(3))))
    for b in range(2):
        got = {k: np.concatenate([p[b][k] for p in parts]) for k in ("state", "pose", "map_to_odom", "map_published")}
        got["maps"] = [m for p in parts for m in p[b]["maps"]]
        assert_same_node(snapshot(fleet.mapper(b), got), wants[b], names[b])
    fleet.close()
