"""Generate tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref/libkarto_ref.so, asserts enabled).

Needs the reference build (`python -m oracle.recipes --ref <checkout of the original project>`):
    python tests/golden/make_golden.py
The answers the *_live tests record (tests/golden/reference/) are rewritten by running those tests with
SLAM_RECORD_GOLDEN=1 where the reference build is present.
The vectors pin the C restatement (oracle/karto_oracle.c) and, through it, the CUDA path.
Every array is produced by the reference's own code; this script only chooses inputs.
"""
import hashlib
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("creating-2d-laser-slam-from-scratch_b200")
synth = pkg.synth
from oracle import ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
D = ref.KT_PI_180


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def small_case():
    """Full dumps on a small problem: Sick LMS200 preset (361 beams, 0.5 deg), 11x11 cell search space."""
    laser = synth.Laser(type=2, n_readings=361, min_angle=synth.deg2rad(-90), max_angle=synth.deg2rad(90),
                        angular_resolution=synth.deg2rad(0.5), min_range=0.0, max_range=80.0, range_threshold=6.0)
    out = {}
    for tag, dropout in (("clean", 0.0), ("dropout", 0.03)):
        mc = synth.make_match_case(11 if dropout == 0 else 12, laser, dropout=dropout, max_xy=0.15, max_th_deg=5)
        p = ref.default_matcher_params(0.5, 0.05, 0.03, 6.0)
        s = ref.RefSession(p, laser)
        assert s.n_readings == 361
        b = s.add_scan(mc.base_ranges, mc.base_pose)
        c = s.add_scan(mc.ranges, mc.odom_pose)
        s.set_grid_from_scans(c, [b])
        gi = s.grid_info()
        sp = s.sensor_pose(c)
        A, R = 10 * D, 1 * D
        out.update({
            f"{tag}_base_ranges": mc.base_ranges, f"{tag}_base_pose": mc.base_pose, f"{tag}_ranges": mc.ranges,
            f"{tag}_pose": mc.odom_pose, f"{tag}_grid": s.grid(), f"{tag}_grid_offset": gi["offset"],
            f"{tag}_grid_info": np.array([gi[k] for k in ("width", "height", "width_step", "data_size", "roi_x",
                                                         "roi_y", "roi_w", "roi_h", "kernel_size")], np.int32),
            f"{tag}_kernel": s.kernel(), f"{tag}_points": s.point_readings(c),
            f"{tag}_valid_points_base": s.find_valid_points(b, sp[:2]),
            f"{tag}_lut": s.compute_offsets(c, sp[2], A, R),
            f"{tag}_sums": s.response_sums(c, sp, (0.25, 0.25), (0.05, 0.05), A, R),
        })
        for pen in (0, 1):
            r = s.correlate_scan(c, sp, (0.25, 0.25), (0.05, 0.05), A, R, do_penalize=bool(pen), fine=False)
            out[f"{tag}_corr_pen{pen}"] = np.concatenate([[r[0]], r[1], r[2].ravel()])
            rf = s.correlate_scan(c, r[1], (0.05, 0.05), (0.05, 0.05), 1 * D, 0.2 * D, do_penalize=bool(pen),
                                  fine=True, cov_in=r[2])
            out[f"{tag}_fine_pen{pen}"] = np.concatenate([[rf[0]], rf[1], rf[2].ravel()])
        m = s.match_scan(c, [b])
        out[f"{tag}_match"] = np.concatenate([[m[0]], m[1], m[2].ravel()])
        og = s.occupancy_grid([b, c], 0.05)
        out[f"{tag}_occ_dims"] = np.array([og["width"], og["height"], og["width_step"]], np.int32)
        out[f"{tag}_occ_offset"] = og["offset"]
        out[f"{tag}_occ_pass"] = og["passes"]
        out[f"{tag}_occ_hit"] = og["hits"]
        out[f"{tag}_occ_cells"] = og["cells"]
        s.close()
    np.savez_compressed(os.path.join(HERE, "karto_small.npz"), **out)


def cfg1_case():
    """BASELINE cfg 1: Hokuyo UTM-30LX (1081 beams), 31x31x181 direct CorrelateScan; digests + results."""
    out = {}
    laser = synth.Laser()
    A, R = 22.5 * D, 0.25 * D
    for seed in range(4):
        mc = synth.make_match_case(seed, laser, dropout=0.01 if seed == 3 else 0.0)
        p = ref.default_matcher_params(1.5, 0.05, 0.03, 9.25)
        s = ref.RefSession(p, laser)
        b = s.add_scan(mc.base_ranges, mc.base_pose)
        c = s.add_scan(mc.ranges, mc.odom_pose)
        s.set_grid_from_scans(c, [b])
        sp = s.sensor_pose(c)
        grid, lut = s.grid(), s.compute_offsets(c, sp[2], A, R)
        sums = s.response_sums(c, sp, (0.75, 0.75), (0.05, 0.05), A, R)
        r = s.correlate_scan(c, sp, (0.75, 0.75), (0.05, 0.05), A, R, True, False)
        m = s.match_scan(c, [b])
        t = f"s{seed}"
        out.update({
            f"{t}_base_ranges": mc.base_ranges, f"{t}_base_pose": mc.base_pose, f"{t}_ranges": mc.ranges,
            f"{t}_pose": mc.odom_pose, f"{t}_grid_sha": np.array(sha(grid)), f"{t}_lut_sha": np.array(sha(lut)),
            f"{t}_sums_sha": np.array(sha(sums)), f"{t}_sums_max_per_angle": sums.max(axis=(0, 1)),
            f"{t}_sums_center_plane": sums[:, :, 90].copy(), f"{t}_grid_nonzero": np.array(int((grid > 0).sum())),
            f"{t}_corr": np.concatenate([[r[0]], r[1], r[2].ravel()]),
            f"{t}_match": np.concatenate([[m[0]], m[1], m[2].ravel()]),
        })
        s.close()
    np.savez_compressed(os.path.join(HERE, "karto_cfg1.npz"), **out)


def multi_base_case():
    """AddScans with 12 base scans along a short trajectory + Karto occupancy grid of all of them; custom laser
    (exercises the 'no +1' beam-count quirk, Karto.h:4158-4160: -90..90 @1deg -> 180 beams)."""
    laser = synth.Laser(type=0, n_readings=180, min_angle=synth.deg2rad(-90), max_angle=synth.deg2rad(90),
                        angular_resolution=synth.deg2rad(1.0), min_range=0.05, max_range=25.0, range_threshold=8.0,
                        offset_pose=(0.12, -0.03, 0.05))
    world, poses, ranges = synth.make_trajectory(5, 13, laser, step_xy=0.2, step_th_deg=4.0)
    p = ref.default_matcher_params(0.8, 0.1, 0.1, 8.0, use_response_expansion=1)
    s = ref.RefSession(p, laser)
    assert s.n_readings == 180, s.n_readings
    ids = [s.add_scan(ranges[i], poses[i]) for i in range(13)]
    odom = poses[12] + np.array([0.11, -0.07, 0.04])
    s.set_pose(ids[12], odom)
    m = s.match_scan(ids[12], ids[:12])
    gi = s.grid_info()
    og = s.occupancy_grid(ids, 0.1)
    np.savez_compressed(os.path.join(HERE, "karto_multibase.npz"), ranges=ranges, poses=poses, odom=odom,
                        grid=s.grid(), grid_offset=gi["offset"], match=np.concatenate([[m[0]], m[1], m[2].ravel()]),
                        sensor_pose=s.sensor_pose(ids[12]),
                        occ_dims=np.array([og["width"], og["height"], og["width_step"]], np.int32),
                        occ_offset=og["offset"], occ_pass=og["passes"], occ_hit=og["hits"], occ_cells=og["cells"])
    s.close()


def trace_lines():
    rng = np.random.default_rng(42)
    segs = rng.integers(-8, 72, size=(400, 4)).astype(np.int32)
    cells, lens = [], []
    for x0, y0, x1, y1 in segs:
        c = ref.trace_line(64, 48, int(x0), int(y0), int(x1), int(y1))
        cells.append(c)
        lens.append(len(c))
    np.savez_compressed(os.path.join(HERE, "karto_tracelines.npz"), segs=segs, lens=np.array(lens, np.int32),
                        cells=np.concatenate(cells).astype(np.int16))


def gmapping_case():
    """lesson4 GMapping ComputeMap through the reference's real grid headers (oracle/ref_gmapping.cpp)."""
    from oracle import ref_gmapping as rg
    laser = synth.Laser()
    out = {}
    # the node computes beam angles in float32 (angle_min + i * angle_increment are float32 message fields)
    ang = (np.float32(laser.min_angle) + np.arange(1081, dtype=np.float32) * np.float32(laser.angular_resolution))
    out["angles"] = ang.astype(np.float64)
    for k, (seed, bounds, lxy) in enumerate([(3, (-40.0, -40.0, 40.0, 40.0, 0.05), (0.0, 0.0)),
                                             (4, (-20.0, -20.0, 30.1, 29.9, 0.05), (1.3, -0.7))]):
        mc = synth.make_match_case(seed, dropout=0.02)
        r = mc.ranges.astype(np.float32).astype(np.float64)  # LaserScan.ranges are float32
        r[5], r[9], r[11] = 0.0, 28.0, 35.0
        m = rg.RefGMap(*bounds)
        assert m.compute_map(r, out["angles"], lxy) == 0
        n, v, ax, ay, occ = m.cells()
        ys, xs = np.nonzero(v)
        out.update({f"c{k}_ranges": r, f"c{k}_bounds": np.array(bounds), f"c{k}_laser_xy": np.array(lxy),
                    f"c{k}_size": np.array([m.size_x, m.size_y], np.int32),
                    f"c{k}_cells_yx": np.stack([ys, xs], 1).astype(np.int16), f"c{k}_n": n[ys, xs], f"c{k}_visits": v[ys, xs],
                    f"c{k}_acc_x": ax[ys, xs], f"c{k}_acc_y": ay[ys, xs]})
        m.close()
    np.savez_compressed(os.path.join(HERE, "gmapping.npz"), **out)


def hector_case():
    """lesson4 HectorSlamProcessor (3-level MapRepMultiMap: GN match + log-odds update) and updateByScanJustOnce through
    the reference's real headers (oracle/ref_hector.cpp; Eigen stand-in oracle/shim/Eigen/mini_eigen.h)."""
    from oracle import ref_hector as rh
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_hector_reference import data_container
    laser = synth.Laser(n_readings=541, angular_resolution=synth.deg2rad(0.5))  # every other beam keeps the file small
    n = 14
    _, poses, ranges = synth.make_trajectory(41, n, laser, step_xy=0.15, step_th_deg=3.0)
    kw = dict(resolution=0.05, size_x=640, size_y=640, start=(0.5, 0.5), levels=3, min_dist=0.12, min_angle=0.05)
    p = rh.RefHectorProcessor(**kw)
    out = {"resolution": np.float32(0.05), "size": np.int32(640), "min_dist": np.float32(0.12), "min_angle": np.float32(0.05),
           "n_scans": np.int32(n), "start_pose": poses[0].astype(np.float32),
           "without_matching": np.array([1] + [0] * (n - 1), np.int8)}
    est, trace = poses[0].astype(np.float32), []
    for i in range(n):
        pts = data_container(laser, ranges[i]).astype(np.float32)
        out[f"pts{i}"] = pts
        est, cov = p.update(pts, (0, 0), est, i == 0)
        trace.append(np.concatenate([est, cov.ravel()]))
    out["trace"] = np.array(trace, np.float32)
    for lvl in range(3):
        lo, ui = p.level(lvl)
        idx = np.flatnonzero(ui.ravel() >= 0)
        out[f"l{lvl}_idx"], out[f"l{lvl}_ui"], out[f"l{lvl}_lo"] = idx, ui.ravel()[idx], lo.ravel()[idx]
    assert (out["l0_ui"].max() + 1) // 3 >= 4
    rng = np.random.default_rng(77)
    jo = rng.uniform(-12, 12, (300, 2)).astype(np.float32)
    m = rh.RefHectorMap(1601, 1601, 0.05)
    m.update_by_scan_just_once(jo, (0, 0))
    lo, ui = m.cells()
    idx = np.flatnonzero(ui.ravel() >= 0)
    out.update({"jo_size": np.int32(1601), "jo_pts": jo, "jo_idx": idx, "jo_ui": ui.ravel()[idx], "jo_lo": lo.ravel()[idx]})
    np.savez_compressed(os.path.join(HERE, "hector.npz"), **out)


def mapper_case():
    """The whole lesson6 front end: karto::Mapper::Process over a seeded 150-scan, 3-lap workload (tests/mapper_cases.py);
    poses and graph edges as the reference leaves them (no back end)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mapper_cases as mc
    seed, n = 3, 150
    laser, prm, true, odom, ranges = mc.workload(pkg, seed, n)
    r = ref.RefMapper(prm, laser)
    flags, _ = mc.run(r, odom, ranges)
    ids, diff, cov = r.edges()
    np.savez_compressed(os.path.join(HERE, "karto_mapper.npz"), seed=np.int32(seed), n=np.int32(n), flags=flags,
                        poses=r.poses(), edge_ids=ids, edge_diff=diff, edge_cov=cov, ranges_sample=ranges[::17])
    r.close()


def fleet_case():
    """Three sensors (robots) feeding one karto::Mapper (MapperSensorManager, Mapper.cpp:45-100, 920-952): poses in
    unique-id order and graph edges as the reference leaves them."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mapper_cases as mc
    seed, n = 3, 150
    laser, prm, true, odom, ranges = mc.workload(pkg, seed, n, drift=mc.FLEET_DRIFT)
    r = ref.RefMapper(prm, laser)
    sensors = [0, r.add_sensor("a_robot"), r.add_sensor("z_robot")]
    flags, _ = mc.run_fleet(r, sensors, odom, ranges)
    ids, diff, cov = r.edges()
    np.savez_compressed(os.path.join(HERE, "karto_mapper_fleet.npz"), seed=np.int32(seed), n=np.int32(n), flags=flags,
                        poses=r.poses_by_id(), edge_ids=ids, edge_diff=diff, edge_cov=cov, ranges_sample=ranges[::17])
    r.close()


if __name__ == "__main__":
    assert ref.available(), "run `python -m oracle.recipes --ref <checkout>` first"
    if sys.argv[1:] == ["mapper"]:
        mapper_case()
        print("karto_mapper.npz", os.path.getsize(os.path.join(HERE, "karto_mapper.npz")))
        sys.exit(0)
    if sys.argv[1:] == ["fleet"]:
        fleet_case()
        print("karto_mapper_fleet.npz", os.path.getsize(os.path.join(HERE, "karto_mapper_fleet.npz")))
        sys.exit(0)
    if sys.argv[1:] == ["hector"]:
        hector_case()
        print("hector.npz", os.path.getsize(os.path.join(HERE, "hector.npz")))
        sys.exit(0)
    small_case()
    cfg1_case()
    multi_base_case()
    trace_lines()
    gmapping_case()
    hector_case()
    mapper_case()
    fleet_case()
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(HERE, f)))
