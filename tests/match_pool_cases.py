"""Workloads that drive the Karto Mapper's shared match pool (MatchPool, csrc/karto_mapper.cu) to its capacity edges,
and a recorder of the match requests a Mapper sends, for tests/test_match_pool_premises.py (CPU) and
tests/test_gpu_match_pool.py (H100).

A MatchPool keeps two b2s_matcher handles, sequential (which = 0) and loop (which = 1), each created on first use with
room for first_batch(clients) matches and chains of first_base(scan_buffer_size) scans, and re-created (every client's
pool rows dropped) when a group of requests does not fit.  PoolModel restates that rule, so a premise can name the
request at which a handle is created or grows; the recorded requests come from the Mapper's host logic with the CPU
restatement's MatchScan behind it (oracle.port.mapper_match_hook), which is exactly what the device Mapper sends."""
from __future__ import annotations

import functools
import importlib
import math
from dataclasses import dataclass, field

import numpy as np

from oracle import port

PKG = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
synth, abi = PKG.synth, PKG.abi
MP = PKG.load("mapper")

MATCH_MAX_BATCH = 256  # matches per launch; a larger group goes out in parts


def first_batch(clients):
    return min(max(8, 2 * clients), MATCH_MAX_BATCH)


def first_base(scan_buffer_size):
    return max(32, scan_buffer_size + 1)


class PoolModel:
    """The capacity rule of one MatchPool: serve() -> "create", "grow" or None for a group of `total` matches whose
    longest chain has `max_base` scans on handle `which`."""

    def __init__(self, clients, scan_buffer_size):
        self.first_batch, self.first_base = first_batch(clients), first_base(scan_buffer_size)
        self.cap_batch, self.cap_base = [0, 0], [0, 0]

    def serve(self, which, total, max_base):
        batch = min(total, MATCH_MAX_BATCH)
        if self.cap_batch[which] and batch <= self.cap_batch[which] and max_base <= self.cap_base[which]:
            return None
        event = "grow" if self.cap_batch[which] else "create"
        self.cap_batch[which] = min(max(batch, 2 * self.cap_batch[which], self.first_batch), MATCH_MAX_BATCH)
        self.cap_base[which] = max(max_base, 2 * self.cap_base[which], self.first_base)
        return event


@dataclass
class Request:
    which: int
    batch: int
    n_base: list
    do_penalize: int
    do_refine: int
    scans: int                 # the Mapper's scans when the request was sent: the client's pool rows on that handle
    event: str | None = None   # PoolModel's verdict for this request served alone (a standalone Mapper)
    caps: tuple = ()           # (cap_batch, cap_base) of both handles after the request
    rows_before: tuple = ()    # pool rows the client held on (sequential, loop) before the request

    @property
    def max_base(self):
        return max(self.n_base)


class Recorder:
    """A b2s_match_scan_fn for mapper.Mapper(match_fn=...): records each request, then serves it with the CPU
    restatement's MatchScan.  `mapper` must be set to the Mapper before its first process()."""

    def __init__(self, prm, laser, clients=1):
        self.hook = port.mapper_match_hook(prm, laser)
        self.model = PoolModel(clients, prm.scan_buffer_size)
        self.requests: list[Request] = []
        self.rows = [0, 0]
        self.mapper = None
        self.log = []  # the requests, and whatever else the caller appends between them (a node's map builds)

    def __call__(self, user, which, batch, ranges, poses, base_first, n_base, base_ranges, base_poses, do_penalize,
                 do_refine, results):
        scans = MP._bind().b2s_mapper_scan_count(self.mapper.h)
        q = Request(which, batch, [n_base[b] for b in range(batch)], do_penalize, do_refine, scans)
        q.rows_before = tuple(self.rows)
        q.event = self.model.serve(which, batch, q.max_base)
        if q.event:
            self.rows[which] = 0
        self.rows[which] = scans
        q.caps = (tuple(self.model.cap_batch), tuple(self.model.cap_base))
        self.requests.append(q)
        self.log.append(q)
        return self.hook(user, which, batch, ranges, poses, base_first, n_base, base_ranges, base_poses, do_penalize,
                         do_refine, results)

    def events(self, which=None):
        return [(k, q) for k, q in enumerate(self.requests) if q.event and (which is None or q.which == which)]


# ------------------------------------------------------------------------------------------------ workloads

# tests/mapper_cases.py's laser and windows, the loop matcher's cut to +-2 m, +-10 deg to keep the restatement cheap
LASER = dict(range_threshold=9.25)
KW = dict(scan_buffer_size=20, link_match_minimum_response_fine=0.1, link_scan_maximum_distance=1.5,
          loop_search_maximum_distance=3.0, loop_match_minimum_chain_size=5, loop_match_maximum_variance_coarse=9.0,
          loop_match_minimum_response_coarse=0.35, loop_match_minimum_response_fine=0.45,
          sequential_search_size=0.5, sequential_resolution=0.05, loop_search_size=2.0,
          loop_coarse_search_angle_offset=synth.deg2rad(10.0))


@dataclass
class Workload:
    name: str
    laser: object                 # synth.Laser
    params: object                # mapper.MapperParams
    events: list = field(default_factory=list)   # [(sensor name or None, ranges, odometric pose)]

    @property
    def al(self):
        return abi.laser_from(self.laser)


def _stream(seed, n, step=0.25, **kw):
    laser = synth.Laser(**LASER)
    _, _, odom, ranges = synth.make_loop_trajectory(seed, n, laser, radius=2.0, step=step)
    return laser, MP.default_params(laser.range_threshold, **dict(KW, **kw)), odom, ranges


def batch_growth(sensors=34):
    """`sensors` sensors, 1 cm apart on the circle, each with one scan: the k-th sensor's scan is matched against every
    other sensor's scans in one batch of k - 1 (9, 17 and 33 cross 8, 16 and 32)."""
    laser, prm, odom, ranges = _stream(21, sensors, step=0.01, do_loop_closing=0)
    ev = [("s%02d" % k, ranges[k], odom[k]) for k in range(sensors)]
    return Workload("batch_growth", laser, prm, ev)


CHAIN_JOINS = (31, 32, 33, 66)


def chain_growth():
    """Sensor "a" circles the room; a new sensor joins when "a" holds 31, 32, 33 and 66 scans, so its first scan is
    matched against a chain of that many scans: below, at and one past the first chain capacity (32), then past its
    first doubling (64)."""
    laser, prm, odom, ranges = _stream(22, 72, do_loop_closing=0)
    ev, i = [], 0
    for j, name in zip(CHAIN_JOINS, "bcde"):
        while sum(1 for e in ev if e[0] == "a") < j:
            ev.append(("a", ranges[i], odom[i]))
            i += 1
        ev.append((name, ranges[i], odom[i]))
        i += 1
    return Workload("chain_growth", laser, prm, ev)


def pool_rows(n=530):
    """One sensor, n key frames, no loop closing: the sequential handle's scan pool passes 256 and 512 rows."""
    laser, prm, odom, ranges = _stream(3, n, do_loop_closing=0)
    return Workload("pool_rows", laser, prm, [(None, ranges[i], odom[i]) for i in range(n)])


# key frames every 5 cm, loop candidates up to 3.8 m away and a strict coarse response: the loop chains of the second
# lap grow past 32 scans before a loop closes
DENSE = dict(minimum_travel_distance=0.04, loop_search_maximum_distance=3.8, loop_match_minimum_response_coarse=0.75)


def loop_growth(n=260):
    """A loop-closing stream whose loop handle, created for a short candidate chain, meets a longer one later and is
    re-created while the sequential handle keeps its pool."""
    laser, prm, odom, ranges = _stream(3, n, step=0.05, **DENSE)
    return Workload("loop_growth", laser, prm, [(None, ranges[i], odom[i]) for i in range(n)])


WORKLOADS = {f.__name__: f for f in (batch_growth, chain_growth, pool_rows, loop_growth)}


def run(mapper, wl, dt=0.1):
    """-> (accepted flags, Process's corrected-pose outputs) of every event"""
    flags, outs = [], []
    for k, (sensor, r, o) in enumerate(wl.events):
        ok, c = mapper.process(r, o, dt * k, sensor=sensor)
        flags.append(ok)
        outs.append(c)
    return np.array(flags), np.array(outs)


def recorded(wl):
    """wl through a Mapper served by the restatement behind a Recorder -> (mapper, recorder, flags, outputs)"""
    rec = Recorder(wl.params, wl.al)
    m = MP.Mapper(wl.params, wl.al, match_fn=rec)
    rec.mapper = m
    flags, outs = run(m, wl)
    return m, rec, flags, outs


# ------------------------------------------------------------------------------------------------ node batches

KN = PKG.load("karto_node")
IDENT = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)


def node_params(kc, **kw):
    """karto_node_cases.SMALL with the loop matcher cut to +-2 m and the coarse sweeps to +-10 deg"""
    return dict(kc.SMALL, loop_search_space_dimension=2.0, coarse_search_angle_offset=math.radians(10.0), **kw)


@functools.lru_cache(maxsize=None)
def node_recordings(kc):
    """name -> (ranges float32, stamps, odom rows) on karto_node_cases' laser: "laps", six laps of 25 cm steps whose
    loops close every lap, and "dense", 5 cm steps (with DENSE's host parameters its loop chain outgrows 32 scans)"""
    out = {}
    r, o = kc.recording(4, 300)
    out["laps"] = (r, kc.stamps_10hz(300), kc.odom_rows(o))
    laser = synth.Laser(type=0, n_readings=kc.N_BEAMS, min_angle=float(kc.ANGLE_MIN),
                        max_angle=float(kc.ANGLE_MIN + kc.N_BEAMS * kc.ANGLE_INC), angular_resolution=float(kc.ANGLE_INC),
                        range_threshold=9.25)
    _, _, o, r = synth.make_loop_trajectory(3, 260, laser, radius=2.0, step=0.05)
    out["dense"] = (r.astype(np.float32), kc.stamps_10hz(260), kc.odom_rows(o))
    return out


def node_trace(params, geometry, ranges, stamps, odom):
    """One SlamKarto node's device requests in order, its Mapper served by the restatement: Request for a match batch,
    "map" for a map build (the map itself is not built).  Round k of a node batch holds each live node's k-th entry.
    -> (requests, ends): the node on the first S scans sends requests[:ends[S - 1]]."""
    from oracle import karto_node_port
    prm, _ = KN.node_params(params)
    node = karto_node_port.PortKartoNode(prm, geometry, IDENT)
    node.mapper.close()
    rec = Recorder(prm.mapper, node.laser)
    node.mapper = rec.mapper = MP.Mapper(prm.mapper, node.laser, match_fn=rec)
    node.update_map = lambda: (rec.log.append("map"), ({}, None))[1]
    ends = []
    for i in range(len(ranges)):
        node.process(ranges[i:i + 1], stamps[i:i + 1], odom[i:i + 1])
        ends.append(len(rec.log))
    node.close()
    return rec.log, ends


def simulate_batch(traces, window):
    """The rounds of one node-batch call over traces[b] (node_trace's), served by one MatchPool: -> dict(launches,
    matches, straddles=[(round, node)] whose batch spans two launches, regrowth=[(round, node, others)] where the loop
    handle is re-created for `node` while `others` (not in that group) hold rows on it, later=[nodes among those
    others that send a loop request after the re-creation])"""
    model = PoolModel(len(traces), window)
    holders = [set(), set()]
    out = dict(launches=0, matches=0, straddles=[], regrowth=[], later=set())
    grown_at = None
    for r in range(max(len(t) for t in traces)):
        groups = {}
        for b, t in enumerate(traces):
            if r < len(t) and t[r] != "map":
                q = t[r]
                groups.setdefault((q.which, q.do_penalize, q.do_refine), []).append((b, q))
        for (which, _, _), g in groups.items():
            total, max_base = sum(q.batch for _, q in g), max(q.max_base for _, q in g)
            clients = {b for b, _ in g}
            if which == 1 and grown_at is not None:
                out["later"] |= clients & grown_at
            event = model.serve(which, total, max_base)
            if event == "grow" and which == 1 and holders[1] - clients:
                grown = max(g, key=lambda x: x[1].max_base)[0]
                out["regrowth"].append((r, grown, sorted(holders[1] - clients)))
                grown_at = holders[1] - clients
            if event:
                holders[which] = set()
            holders[which] |= clients
            cap = model.cap_batch[which]
            out["launches"] += -(-total // cap)
            out["matches"] += total
            t = 0
            for b, q in g:
                if total > cap and t // cap != (t + q.batch - 1) // cap:
                    out["straddles"].append((r, b))
                t += q.batch
    out["later"] = sorted(out["later"])
    return out


def straddle_nodes(kc, S, B=300, seed=300):
    """B nodes on node_recordings' "laps" (S scans): throttle 1, 2 or 3 and a prefix of it, every fourth node at full
    length -> [(params, length)]"""
    rng = np.random.default_rng(seed)
    return [(node_params(kc, map_update_interval=1.0, throttle_scans=1 + b % 3),
             S if b % 4 == 0 else int(rng.integers(S // 2, S + 1))) for b in range(B)]
