"""The workloads of tests/test_gpu_match_pool.py reach the match pool's capacity edges (tests/match_pool_cases.py).

Each workload runs through the Mapper's host logic with the CPU restatement's MatchScan behind a request recorder, and
the recorded requests are checked against the pool's capacity rule: if a workload drifts off the edge it exists for,
this file fails, not silently the GPU test that relies on it.  No GPU here."""
import functools

import karto_node_cases as kc
import match_pool_cases as mc


@functools.lru_cache(maxsize=None)
def recorded(name):
    m, rec, flags, _ = mc.recorded(mc.WORKLOADS[name]())
    stats = m.stats()
    m.close()
    return rec, flags, stats


def test_capacity_model():
    """the rule as karto_mapper.cu states it: first capacities, doubling, the 256-match batch limit"""
    assert (mc.first_batch(1), mc.first_batch(4), mc.first_batch(132), mc.first_batch(300)) == (8, 8, 256, 256)
    assert (mc.first_base(20), mc.first_base(31), mc.first_base(110)) == (32, 32, 111)
    p = mc.PoolModel(1, 20)
    assert p.serve(0, 1, 20) == "create" and (p.cap_batch[0], p.cap_base[0]) == (8, 32)
    assert p.serve(0, 8, 32) is None
    assert p.serve(0, 9, 1) == "grow" and (p.cap_batch[0], p.cap_base[0]) == (16, 64)
    assert p.serve(0, 3, 200) == "grow" and (p.cap_batch[0], p.cap_base[0]) == (32, 200)
    assert p.serve(0, 1000, 1) == "grow" and p.cap_batch[0] == 256
    assert p.serve(0, 1000, 1) is None  # a group of 1000 goes out in four launches of at most 256
    assert p.cap_batch[1] == 0 and p.serve(1, 1, 40) == "create" and p.cap_base[1] == 40


def test_batch_growth_crosses_8_16_32():
    rec, flags, _ = recorded("batch_growth")
    assert flags.all()
    grows = [(q.batch, q.caps[0][0]) for _, q in rec.events(0)]
    assert grows == [(1, 8), (9, 16), (17, 32), (33, 64)], grows
    assert max(q.max_base for q in rec.requests) == 1  # every other sensor holds one scan


def test_chain_growth_reaches_the_first_capacity_and_passes_it_twice():
    rec, flags, _ = recorded("chain_growth")
    assert flags.all()
    first = [q for q in rec.requests if q.batch > 1 or q.max_base > 20]  # the joining sensors' batches
    assert [q.max_base for q in first][-3:] == [32, 33, 66], [q.max_base for q in first]
    at_cap = next(q for q in first if q.max_base == 32)
    assert at_cap.event is None and at_cap.caps[1][0] == 32  # exactly the first chain capacity: no re-creation
    grows = [(q.max_base, q.caps[1][0], q.rows_before[0]) for _, q in rec.events(0)][1:]
    assert [g[:2] for g in grows] == [(33, 64), (66, 128)], grows
    assert all(g[2] > 32 for g in grows)  # the handle held pool rows when it was re-created


def test_pool_rows_pass_256_and_512():
    rec, flags, stats = recorded("pool_rows")
    assert flags.all() and stats["loops_closed"] == 0
    assert [e for e in rec.events()] == [(0, rec.requests[0])]  # one sequential handle, never re-created
    assert max(q.scans for q in rec.requests) > 520 and any(q.scans == 256 for q in rec.requests)
    assert any(q.scans == 512 for q in rec.requests)


def test_loop_handle_grows_while_the_sequential_handle_keeps_its_rows():
    rec, flags, stats = recorded("loop_growth")
    ev = [(k, q.which, q.event) for k, q in rec.events()]
    assert [e[1:] for e in ev][:3] == [(0, "create"), (1, "create"), (1, "grow")], ev
    k, q = rec.events(1)[1]
    assert q.max_base > 32 and q.caps[1][1] == 64 and q.rows_before[1] > 0 and q.rows_before[0] > 200
    assert any(r.which == 0 for r in rec.requests[k + 1:]) and any(r.which == 1 for r in rec.requests[k + 1:])
    assert stats["loops_closed"] >= 1


@functools.lru_cache(maxsize=None)
def node_trace(name, throttle=1):
    recs = mc.node_recordings(kc)
    extra = mc.DENSE if name == "dense" else {}
    if name == "loops_small_windows":
        c = kc.CASES[name]
        rows = (c.ranges, c.stamps, c.odom)
    else:
        rows = recs[name]
    p = mc.node_params(kc, map_update_interval=1.0, throttle_scans=throttle, **extra)
    return mc.node_trace(p, kc.CASES["loops_small_windows"].geometry(), *rows)


def test_node_batch_of_300_splits_every_group():
    log, ends = node_trace("loops_small_windows")
    sim = mc.simulate_batch([log] * 300, 20)
    one = mc.simulate_batch([log], 20)
    assert sim["matches"] == 300 * one["matches"] and sim["launches"] >= 2 * one["launches"]


def straddle_traces():
    out = []
    for p, S in mc.straddle_nodes(kc, len(mc.node_recordings(kc)["laps"][0])):
        log, ends = node_trace("laps", p["throttle_scans"])
        out.append(log[:ends[S - 1]])
    return out


def test_node_requests_straddle_the_256_boundary():
    sim = mc.simulate_batch(straddle_traces(), 20)
    assert len(sim["straddles"]) >= 3, sim["straddles"]
    assert sim["launches"] > len({r for r, _ in sim["straddles"]})


def test_node_loop_chain_outgrows_the_first_capacity_mid_call():
    """the "dense" node's loop chain passes 32 scans while the "laps" node holds rows on the loop handle, and the
    "laps" node sends loop requests after that"""
    sim = mc.simulate_batch([node_trace("laps")[0], node_trace("dense")[0]], 20)
    assert [(g[1], g[2]) for g in sim["regrowth"]] == [(1, [0])], sim["regrowth"]
    assert sim["later"] == [0]
