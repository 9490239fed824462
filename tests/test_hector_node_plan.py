"""hector_node_plan (csrc/hector_node_plan.cuh) decides on the host where every node of a b2s_hector_node handle
publishes in a call and how the call splits into launches.  tests/hector_node_plan_check.cu runs it without a GPU.
Checked here, node by node, against the restatement's schedule (oracle/hector_node_port.Schedule), over the recordings
of hector_node_cases, exact ticks and seeded random batches with gaps, empty nodes and continuation calls: the publish
points and ticks, the schedule carried to the next call, and the parts (each node's scans in exactly one part, in order,
part k >= 1 starting at the node's k-th publish, 1 + the largest publish count parts)."""
import importlib
import json
import os
import subprocess

import numpy as np
import pytest

import hector_node_cases as cases
from oracle import hector_node_port as P

HERE = os.path.dirname(os.path.abspath(__file__))
NS = 1_000_000_000


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    exe = str(tmp_path_factory.mktemp("hector_node_plan") / "hector_node_plan_check")
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           os.path.join(HERE, "hector_node_plan_check.cu"), "-o", exe])

    def run(requests):
        """requests: [[(clock (started, next_tick_ns), period_ns, stamps [n][2]) per node]] -> one dict per request"""
        lines = []
        for nodes in requests:
            words = [str(len(nodes))]
            for (started, nxt), period, st in nodes:
                st = np.asarray(st, np.uint32).reshape(-1, 2)
                words += [str(int(started)), str(int(nxt)), str(int(period)), str(len(st))]
                words += [str(int(v)) for v in st.reshape(-1)]
            lines.append(" ".join(words) + "\n")
        out = subprocess.run([exe], input="".join(lines), capture_output=True, text=True, check=True)
        return [json.loads(line) for line in out.stdout.splitlines()]

    return run


def period_ns(seconds):
    sec, nsec = P.duration_from_sec(seconds)
    return sec * NS + nsec


class Node:
    """One node's schedule over calls: the restatement's, and the clock the plan carries."""

    def __init__(self, period):
        self.period = period
        self.schedule = P.Schedule(period)
        self.clock = (0, 0)

    def expect(self, stamps):
        cuts, ticks = [], []
        for i, s in enumerate(np.asarray(stamps, np.uint32).reshape(-1, 2)):
            t = self.schedule.before(s)
            if t is not None:
                cuts.append(i)
                ticks.append(t[0] * NS + t[1])
        return cuts, ticks


def check_call(plan, nodes, calls):
    """nodes: [Node]; calls: [[stamps of node b] per call].  Runs every call through the plan, carrying the clocks."""
    for stamps in calls:
        (r,) = plan([[(n.clock, period_ns(n.period), s) for n, s in zip(nodes, stamps)]])
        most = 0
        for b, (n, s, got) in enumerate(zip(nodes, stamps, r["nodes"])):
            cuts, ticks = n.expect(s)
            assert (got["cuts"], got["ticks"]) == (cuts, ticks), (b, got, cuts, ticks)
            most = max(most, len(cuts))
            # the schedule carried to the next call: the restatement's next tick, once a scan has been seen
            if n.schedule.next is not None:
                assert got["started"] == 1
                assert got["next_tick"] == n.schedule.next[0] * NS + n.schedule.next[1], b
            else:
                assert got["started"] == 0
            n.clock = (got["started"], got["next_tick"])
            # every scan in exactly one part, in order; part k >= 1 starts at the k-th publish
            parts = got["parts"]
            assert len(parts) == r["n_parts"]
            assert parts[0][0] == 0 and parts[-1][1] == len(s)
            for k in range(1, len(parts)):
                assert parts[k][0] == parts[k - 1][1], (b, parts)
                if k <= len(cuts):
                    assert parts[k][0] == cuts[k - 1], (b, k, parts, cuts)
                else:
                    assert parts[k][0] == parts[k][1] == len(s), (b, k, parts)
            assert all(lo <= hi for lo, hi in parts)
        assert r["n_parts"] == 1 + most


def test_the_node_cases(plan):
    cs = cases.cases()
    for name, c in sorted(cs.items()):
        check_call(plan, [Node(cases.hector_node.node_params(c["params"]).map_pub_period)], [[c["stamps"]]])
    # all eleven side by side, in one call and in three

    def nodes():
        return [Node(cases.hector_node.node_params(c["params"]).map_pub_period) for _, c in sorted(cs.items())]
    stamps = [c["stamps"] for _, c in sorted(cs.items())]
    check_call(plan, nodes(), [stamps])
    check_call(plan, nodes(), [[s[:2] for s in stamps], [s[2:5] for s in stamps], [s[5:] for s in stamps]])


def test_exact_tick_stamps(plan):
    st = cases.exact_tick_stamps()
    check_call(plan, [Node(0.3)], [[st]])
    check_call(plan, [Node(0.3), Node(0.1), Node(1e6)], [[st, st, st]])
    check_call(plan, [Node(0.3)], [[st[:2]], [st[2:]]])


def random_batch(rng, B):
    nodes, recordings = [], []
    for _ in range(B):
        nodes.append(Node(float(rng.choice([0.01, 0.025, 0.05, 0.1, 0.3, 1.0, 2.0, 1e6]))))
        n = int(rng.integers(0, 60))
        t = int(rng.integers(0, 50)) * NS + int(rng.integers(0, NS))
        dt = int(rng.choice([25_000_000, 10_000_000, 100_000_000, 50_000_000]))
        out = []
        for _ in range(n):
            out.append((t // NS, t % NS))
            r = rng.random()
            t += dt if r > 0.15 else (int(rng.integers(1, 8)) * NS if r > 0.05 else 0)  # gaps, repeated stamps
        recordings.append(np.array(out, np.uint32).reshape(-1, 2))
    return nodes, recordings


def split(rng, recordings, calls):
    """the recordings over `calls` calls: each node cut at its own points, some calls empty for some nodes"""
    edges = [np.sort(np.concatenate([[0], rng.integers(0, len(r) + 1, calls - 1), [len(r)]])) for r in recordings]
    return [[r[e[c]:e[c + 1]] for r, e in zip(recordings, edges)] for c in range(calls)]


@pytest.mark.parametrize("seed", range(12))
def test_random_batches(plan, seed):
    rng = np.random.default_rng(20261016 + seed)
    B = int(rng.integers(1, 40))
    nodes, recordings = random_batch(rng, B)
    check_call(plan, nodes, [recordings])
    # the same recordings in continuation calls give the same publishes
    rng2 = np.random.default_rng(seed)
    nodes2 = [Node(n.period) for n in nodes]
    check_call(plan, nodes2, split(rng2, recordings, int(rng2.integers(2, 6))))


def test_period_ticks_on_stamps(plan):
    """a stamp exactly on the next tick publishes; one a nanosecond before does not"""
    per = period_ns(0.3)
    t0 = 10 * NS
    st = np.array([(10, 0), ((t0 + per - 1) // NS, (t0 + per - 1) % NS), ((t0 + per) // NS, (t0 + per) % NS)], np.uint32)
    (r,) = plan([[((0, 0), per, st)]])
    assert r["nodes"][0]["cuts"] == [0, 2] and r["nodes"][0]["ticks"] == [t0, t0 + per]
    assert r["n_parts"] == 3 and r["nodes"][0]["parts"] == [[0, 0], [0, 2], [2, 3]]
