"""GPU tests of b2s_hector_node_create_fleet and b2s_hector_slam_create_fleet: nodes and processors of different robots
(own laser, own map size / resolution / levels / start / update factors / gate) in one handle.  Every node must equal,
bit for bit, its own single-node handle (and the restatement oracle/hector_node_port.py for the recorded cases): poses,
pose messages, covariances, gate flags, kept-beam counts and every map's payload, info, stamp, scan_index and rebuilt
flag.  Every fleet processor must equal a one-processor handle with the same spec, in exact and in fast mode."""
import numpy as np
import pytest

import hector_node_cases as cases
from test_gpu_hector_node import _assert_maps, _assert_scans, _geom, _node, _port, _same_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
CASES = cases.cases()
SHARED = ["yaw_pi", "upside_down", "pitched_z_window", "bad_ranges", "empty_scans", "schedule_gaps", "short_period"]


@pytest.fixture(scope="module")
def N(pkg):
    assert pkg.load("matcher").device_count() > 0
    return pkg.load("hector_node")


@pytest.fixture(scope="module")
def R(pkg):
    return pkg.load("rosio")


@pytest.fixture(scope="module")
def H(pkg):
    return pkg.load("hector")


@pytest.fixture(scope="module")
def synth(pkg):
    return pkg.synth


def _fleet(N, R, cs):
    return N.HectorNodeBatch.fleet([N.node_params(c["params"]) for c in cs],
                                   [_geom(R, c["geometry"], c["ranges"].shape[1]) for c in cs], [c["mount"] for c in cs])


def _single(N, R, c):
    g = _node(N, R, c)
    out = g.process(c["ranges"], c["stamps"])
    g.close()
    return out


def _each_equals_single(N, R, cs, got):
    for b, c in enumerate(cs):
        if len(c["stamps"]) == 0:
            assert len(got[b]["pose"]) == 0 and not got[b]["maps"]
            continue
        want = _single(N, R, c)
        _assert_scans(got[b], want, b)
        _assert_maps(got[b]["maps"], want["maps"], b)


def test_every_recorded_case_in_one_fleet(N, R):
    """2048^2 and 512^2 maps, the boundary geometry and the rare gate side by side: no create_batch can hold them."""
    names = sorted(CASES)
    cs = [CASES[n] for n in names]
    h = _fleet(N, R, cs)
    got = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    for b, (name, c) in enumerate(zip(names, cs)):
        want = _single(N, R, c)
        _assert_scans(got[b], want, name)
        _assert_maps(got[b]["maps"], want["maps"], name)
        port = _port(N, c)
        pw = port.process(c["ranges"], c["stamps"])
        _assert_scans(got[b], pw, name)
        _assert_maps(got[b]["maps"], pw["maps"], name)
        assert np.array_equal(h.level_ros(b), port.publish_map((0, 0))["payload"]), name
        port.close()
    h.close()


# (beams, field of view in degrees, range_min, range_max): Hokuyo-, 2D-lidar- and dense-scanner-like lasers
LASERS = [(360, 360.0, 0.15, 12.0), (720, 360.0, 0.12, 16.0), (1081, 270.0, 0.1, 30.0), (1440, 360.0, 0.2, 25.0),
          (4096, 360.0, 0.1, 20.0), (1081, 360.0, 0.05, 10.0)]


def _laser(synth, beams, fov, rmin, rmax):
    inc = np.deg2rad(fov) / (beams if fov == 360.0 else beams - 1)
    amin = -np.deg2rad(fov) / 2
    return synth.Laser(n_readings=beams, min_angle=amin, max_angle=amin + inc * (beams - 1), angular_resolution=inc,
                       min_range=rmin, max_range=rmax)


def _mixed(synth, seed, B, max_len=40, sizes=(256, 384, 512, 768, 1024), lasers=LASERS):
    """B walks, each with its own laser, map and schedule (seeded)"""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        beams, fov, rmin, rmax = lasers[int(rng.integers(len(lasers)))]
        las = _laser(synth, beams, fov, rmin, rmax)
        n = int(rng.integers(0, max_len + 1))
        _, _, r = synth.make_trajectory(5000 + 97 * seed + b, max(n, 1), las, step_xy=0.05, step_th_deg=2.0)
        size = int(rng.choice(sizes))
        levels = int(rng.integers(1, 5))
        while (size >> (levels - 1)) <= 2:
            levels -= 1
        params = dict(map_size=size, map_resolution=float(rng.choice([0.025, 0.05, 0.075, 0.1])),
                      map_multi_res_levels=levels, map_start_x=float(rng.uniform(0.3, 0.7)),
                      map_start_y=float(rng.uniform(0.3, 0.7)), update_factor_free=float(rng.choice([0.4, 0.35, 0.45])),
                      update_factor_occupied=float(rng.choice([0.9, 0.7, 0.6])),
                      map_update_distance_thresh=float(rng.choice([0.4, 0.1, 0.02])),
                      map_update_angle_thresh=float(rng.choice([0.9, 0.06, 0.5])),
                      laser_max_dist=float(rng.choice([30.0, 12.0])),
                      map_pub_period=float(rng.choice([0.025, 0.05, 0.1, 0.3, 2.0])))
        st = cases.stamps_at(int(rng.integers(1, 100)), int(rng.integers(0, 1_000_000_000)), 25_000_000, n,
                             gaps=((int(rng.integers(0, max(n, 1))), int(rng.integers(0, 3_000_000_000))),))
        m = cases.mount(float(rng.uniform(-0.1, 0.1)), float(rng.uniform(-0.1, 0.1)), float(rng.uniform(0.0, 0.4)),
                        yaw=float(rng.uniform(-3.1, 3.1)), roll=float(rng.choice([0.0, np.pi])))
        geometry = (f32(las.min_angle), f32(las.angular_resolution), f32(rmin), f32(rmax))
        out.append(dict(params=params, mount=m, geometry=geometry, ranges=r.astype(np.float32)[:n].reshape(n, beams),
                        stamps=st.reshape(n, 2)))
    return out


def test_mixed_fleet_and_chunked_calls(N, R, synth):
    cs = _mixed(synth, 7, 40)
    assert len({c["ranges"].shape[1] for c in cs}) >= 4 and len({c["params"]["map_size"] for c in cs}) >= 4
    h = _fleet(N, R, cs)
    whole = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    _each_equals_single(N, R, cs, whole)
    # three calls, each node cut at its own points (some calls give a node no scans)
    rng = np.random.default_rng(3)
    edges = [np.sort(np.concatenate([[0], rng.integers(0, len(c["stamps"]) + 1, 2), [len(c["stamps"])]])) for c in cs]
    h2 = _fleet(N, R, cs)
    parts = [h2.process([c["ranges"][e[k]:e[k + 1]] for c, e in zip(cs, edges)],
                        [c["stamps"][e[k]:e[k + 1]] for c, e in zip(cs, edges)]) for k in range(3)]
    assert any(e[1] == e[0] or e[2] == e[1] or e[3] == e[2] for e in edges)
    for b in range(len(cs)):
        for key in ("pose", "pose_msg", "cov", "map_updated", "n_points"):
            assert _same_bits(np.concatenate([p[b][key] for p in parts]), whole[b][key]), (b, key)
        _assert_maps([m for p in parts for m in p[b]["maps"]], whole[b]["maps"], b)
    h.close(), h2.close()


def test_more_nodes_than_resident_ctas(N, R, synth):
    cs = _mixed(synth, 11, 270, max_len=16, sizes=(128, 192, 256), lasers=LASERS[:4])
    h = _fleet(N, R, cs)
    got = h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    _each_equals_single(N, R, cs, got)
    h.close()


def test_publish_map_of_each_node_has_its_own_dims(N, R, synth):
    cs = _mixed(synth, 5, 6, max_len=10)
    h = _fleet(N, R, cs)
    h.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    for b, c in enumerate(cs):
        m = h.publish_map(b, (1, 0))
        size, res = c["params"]["map_size"], f32(c["params"]["map_resolution"])
        assert (m["info"]["width"], m["info"]["height"]) == (size, size) and m["payload"].shape == (size, size)
        assert f32(m["info"]["resolution"]) == res
        assert np.array_equal(m["payload"], h.level_ros(b))
        g = _node(N, R, c)
        g.process(c["ranges"], c["stamps"])
        w = g.publish_map((1, 0))
        assert m["info"] == w["info"] and np.array_equal(m["payload"], w["payload"]) and m["rebuilt"] == w["rebuilt"]
        g.close()
    h.close()


def test_equal_fleet_equals_create_batch(N, R):
    cs = [CASES[n] for n in SHARED]
    f = _fleet(N, R, cs)
    b = N.HectorNodeBatch([N.node_params(c["params"]) for c in cs], _geom(R, cs[0]["geometry"], cs[0]["ranges"].shape[1]),
                          [c["mount"] for c in cs])
    gf = f.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    gb = b.process([c["ranges"] for c in cs], [c["stamps"] for c in cs])
    for k in range(len(cs)):
        _assert_scans(gf[k], gb[k], SHARED[k])
        _assert_maps(gf[k]["maps"], gb[k]["maps"], SHARED[k])
    f.close(), b.close()


SPECS = [dict(resolution=0.05, size_x=512, size_y=384, start=(0.5, 0.5), levels=3, update_free=0.4, update_occupied=0.9,
              min_dist=0.1, min_angle=0.06),
         dict(resolution=0.025, size_x=1024, size_y=1024, start=(0.4, 0.6), levels=4, update_free=0.35,
              update_occupied=0.7, min_dist=0.02, min_angle=0.9),
         dict(resolution=0.1, size_x=256, size_y=320, start=(0.5, 0.45), levels=1, update_free=0.45, update_occupied=0.6,
              min_dist=0.4, min_angle=0.13),
         dict(resolution=0.075, size_x=384, size_y=384, start=(0.55, 0.5), levels=2, update_free=0.4,
              update_occupied=0.8, min_dist=0.05, min_angle=0.5)]


def _one(H, s, cap, exact):
    return H.HectorSlam(batch=1, max_points=cap, exact=exact, **s)


def _assert_same_processor(got_h, b, want_h, levels):
    for lv in range(levels):
        assert got_h.level_dims(lv, b) == want_h.level_dims(lv)
        (gl, gu), (wl, wu) = got_h.level_of(b, lv), want_h.level_of(0, lv)
        assert _same_bits(gl, wl) and np.array_equal(gu, wu), (b, lv)
    ga, gu = got_h.last_poses(b)
    wa, wu = want_h.last_poses(0)
    assert _same_bits(ga, wa) and _same_bits(gu, wu), b


@pytest.mark.parametrize("exact", [True, False])
def test_processor_fleet_equals_single_processors(H, R, synth, exact):
    """process_stream_batch and process_scans_batch on a mixed create_fleet handle equal B = 1 create_batch handles
    with the same spec: the same kernel and per-CTA order, so fast mode is bit-equal too."""
    las = synth.Laser()
    specs = [H.map_spec(**s) for s in SPECS]
    streams, rec = [], []
    for b, s in enumerate(SPECS):
        _, _, r = synth.make_trajectory(300 + b, 12 + 3 * b, las, step_xy=0.06, step_th_deg=3.0)
        rec.append(r.astype(np.float32))
        streams.append([H.scan_to_data_container(x, las, s["resolution"]) for x in r])
    f = H.HectorSlam.fleet(specs, max_points=1081, exact=exact)
    assert f.levels == [s["levels"] for s in SPECS]
    with pytest.raises(Exception):
        f.level_dims(1, 2)  # processor 2 has one level
    got, covs = f.process_stream_batch(streams, (0.0, 0.0))
    for b, s in enumerate(SPECS):
        one = _one(H, s, 1081, exact)
        (want,), wc = one.process_stream_batch([streams[b]], (0.0, 0.0))
        assert _same_bits(got[b][0], want[0]) and np.array_equal(got[b][1], want[1]), b
        assert _same_bits(covs[b], wc[0]), b
        _assert_same_processor(f, b, one, s["levels"])
        one.close()
    f.close()
    # raw LaserScans of one laser: each processor scales to its own level-0 cell length
    geom = R.make_msg(f32(las.min_angle), f32(las.max_angle), f32(las.angular_resolution), f32(0.1), f32(30.0),
                      np.zeros(las.n_readings, np.float32))
    f = H.HectorSlam.fleet(specs, max_points=1081, exact=exact)
    got, covs, kept = f.process_scans_batch(geom, rec)
    for b, s in enumerate(SPECS):
        one = _one(H, s, 1081, exact)
        (want,), wc, wk = one.process_scans_batch(geom, [rec[b]])
        assert _same_bits(got[b][0], want[0]) and np.array_equal(got[b][1], want[1]), b
        assert _same_bits(covs[b], wc[0]) and np.array_equal(kept[b], wk[0]), b
        _assert_same_processor(f, b, one, s["levels"])
        one.close()
    f.close()
