"""plan_sweep (csrc/karto_sweep_plan.cuh) decides on the host, before anything is enqueued, which sweep kernel a
CorrelateScan runs, with which candidate stride, row bands and shared-memory sizes, or why the search is refused.
tests/sweep_plan_check.cu runs it without a GPU, for this module and the other test_sweep_plan_* modules.  Checked here: the geometries of the benchmark and of the GPU matcher
tests, every kernel selector, every refusal, and the invariants the kernels rely on over a seeded random sweep."""
import importlib
import json
import math
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
D = math.pi / 180

# The device numbers the plan takes, for an H100: cudaDeviceProp::sharedMemPerBlockOptin (227 KB), the SM count, and
# k_sweep_window's static shared memory as `cuobjdump -res-usage` reports it (SHARED:3200), which is the
# cudaFuncAttributes::sharedSizeBytes the handle reads at create (the 1 KB the driver reserves per block is in neither).
OPTIN = 232_448
SMS = 132
WIN_STATIC = 3_200
LIST_SMEM_MAX = 200 * 1024
WIN_MAX_BANDS = 32
OK, BAD_PARAMS, TOO_LARGE = 0, 1, 7  # B2S_OK, B2S_ERR_BAD_PARAMS, B2S_ERR_TOO_LARGE


@pytest.fixture(scope="session")
def plan(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    exe = str(tmp_path_factory.mktemp("sweep_plan") / "sweep_plan_check")
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           os.path.join(HERE, "sweep_plan_check.cu"), "-o", exe])

    def run(requests):
        out = subprocess.run([exe], input="".join(r + "\n" for r in requests), capture_output=True, text=True, check=True)
        return [json.loads(line) for line in out.stdout.splitlines()]

    return run


def params(search, res, smear, rt):
    return f"{search!r} {res!r} {smear!r} {rt!r}"


def plan_request(p, n, batch, search, k_first=0, na_override=-1, force=0, sat_valid=1, high_bytes=0, optin=OPTIN):
    ox, oy, rx, ry, ao, ar, fine = search
    return (f"plan {p} {n} {batch} {ox!r} {oy!r} {rx!r} {ry!r} {ao!r} {ar!r} {fine} {k_first} {na_override} {force} "
            f"{sat_valid} {high_bytes} {SMS} {optin} {WIN_STATIC}")


def window(side, res, mult=1, angle_offset=10 * D, angle_res=1 * D, fine=0):
    """the full window of the test geometries: Search(half, half, mult * res, mult * res, ...)"""
    half = 0.5 * (side - 1) * res
    return (half, half, mult * res, mult * res, angle_offset, angle_res, fine)


def coarse(side, res, angle_offset=20 * D, angle_res=2 * D):
    """MatchScan's coarse stage (Mapper.cpp:228-234), as b2s_matcher_match_scan forms it"""
    r = 1.0 / (1.0 / res)
    half = 0.5 * (side - 1.0) * r
    return (half, half, 2 * r, 2 * r, angle_offset, angle_res, 0)


def side_of(plan, p):
    return plan([f"layout {p}"])[0]["search_side"]


CFG2 = params(1.5, 0.05, 0.03, 9.25)
CFG2_SEARCH = (0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 0)


def test_cfg2_takes_the_window_kernel_on_the_whole_grid(plan):
    (r,) = plan([plan_request(CFG2, 1081, 1024, CFG2_SEARCH)])
    assert r["status"] == OK and (r["nx"], r["ny"], r["na"]) == (31, 31, 181)
    assert r["use_window"] and r["nbands"] == 1 and r["stride"] == 1 and r["skip_empty"]
    assert not r["need_plain_lut"] and r["ctas"] == SMS


def test_match_scan_coarse_stage_has_stride_2(plan):
    (r,) = plan([plan_request(CFG2, 1081, 1024, coarse(side_of(plan, CFG2), 0.05))])
    assert r["status"] == OK and r["use_window"] and r["stride"] == 2 and r["nbands"] == 1
    assert (r["nx"], r["na"]) == (16, 21)


# the geometries test_gpu_matcher.py sweeps in row bands: (params, search)
BANDED = [
    ("test_other_geometries", params(1.5, 0.025, 0.03, 9.25), lambda side: window(side, 0.025)),
    *[(f"test_banded_window_kernel_large_grids {res} {search} {rt} {na_deg}", params(search, res, 0.03, rt),
       lambda side, res=res, na_deg=na_deg: window(side, res, angle_offset=na_deg * D))
      for res, search, rt, na_deg in [(0.05, 1.5, 12.0, 10), (0.025, 1.5, 9.25, 5), (0.025, 0.75, 9.25, 8),
                                      (0.025, 1.5, 9.25, 4), (0.05, 3.1, 12.0, 4)]],
    ("test_stride2_coarse_lattice rt=50", params(15.0, 0.1, 0.3, 50.0),
     lambda side: window(side, 0.1, mult=2, angle_offset=20 * D, angle_res=2 * D)),
]


@pytest.mark.parametrize("name,p,search", BANDED, ids=[b[0] for b in BANDED])
def test_large_grids_take_the_banded_window_kernel(plan, name, p, search):
    (r,) = plan([plan_request(p, 1081, 3, search(side_of(plan, p)))])
    assert r["status"] == OK and r["use_window"], r
    assert 1 < r["nbands"] <= WIN_MAX_BANDS, r
    assert r["stride"] == (2 if "stride2" in name else 1)


def test_generic_kernel_cases(plan):
    shipped = params(0.3, 0.01, 0.03, 12.0)  # the shipped yaml: 0.01 m, 2431 x 2431 cells inside the border
    side = side_of(plan, shipped)
    reqs = [plan_request(shipped, 1081, 8, window(side, 0.01)),
            plan_request(shipped, 1081, 8, coarse(side, 0.01)),
            plan_request(CFG2, 1081, 8, window(31, 0.05, mult=1.5)),  # neither stride 1 nor 2
            plan_request(CFG2, 1081, 8, CFG2_SEARCH, high_bytes=1),  # a grid byte > 127
            plan_request(CFG2, 8000, 8, CFG2_SEARCH)]  # the list stage's points do not fit in shared memory
    out = plan(reqs)
    assert out[0]["width"] == 2445 and out[0]["nbands"] > WIN_MAX_BANDS
    for r in out:
        assert r["status"] == OK and not r["use_window"] and r["need_plain_lut"], r
    assert out[2]["stride"] == 0


def test_kernel_selectors(plan):
    """b2s_matcher_set_kernel: 0 picks, 1 generic, 2 window, 3 window without empty-window dropping"""
    out = plan([plan_request(CFG2, 1081, 64, CFG2_SEARCH, force=k) for k in range(4)] +
               [plan_request(CFG2, 1081, 64, CFG2_SEARCH, force=k, sat_valid=0) for k in (0, 2)])
    assert [r["use_window"] for r in out[:4]] == [1, 0, 1, 1]
    assert [r["skip_empty"] for r in out] == [1, 1, 1, 0, 0, 0]
    assert out[3]["osm"] < out[2]["osm"] and out[4]["osm"] == out[3]["osm"]


def test_refusals(plan):
    side = side_of(plan, CFG2)
    cases = [
        ((0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.0, 0), {}, BAD_PARAMS, "search resolutions must be non-zero"),
        ((0.75, 0.75, 0.0, 0.05, 22.5 * D, 0.25 * D, 0), {}, BAD_PARAMS, "search resolutions must be non-zero"),
        ((0.75, 0.75, 0.05, 0.0, 22.5 * D, 0.25 * D, 0), {}, BAD_PARAMS, "search resolutions must be non-zero"),
        (CFG2_SEARCH, dict(k_first=-1, na_override=4), BAD_PARAMS, "angle subset outside the search"),
        (CFG2_SEARCH, dict(k_first=178, na_override=4), BAD_PARAMS, "angle subset outside the search"),
        ((40.0, 40.0, 0.05, 0.05, 22.5 * D, 0.25 * D, 0), {}, TOO_LARGE, "search volume too large"),
        ((-0.75, 0.75, 0.05, 0.05, 22.5 * D, 0.25 * D, 0), {}, TOO_LARGE, "search volume too large"),
        (window(side, 0.05, mult=1.5), dict(force=2), TOO_LARGE,
         "window kernel forced but not applicable to this lattice / grid / beam count"),
        (CFG2_SEARCH, dict(force=3, high_bytes=1), TOO_LARGE,
         "window kernel forced but not applicable to this lattice / grid / beam count"),
        (window(side, 0.05, angle_offset=3072 * 0.001, angle_res=0.001, fine=1), {}, TOO_LARGE,
         "too many angles for the angular-covariance kernel"),
    ]
    out = plan([plan_request(CFG2, 1081, 8, s, **kw) for s, kw, _, _ in cases])
    for r, (_, _, status, msg) in zip(out, cases):
        assert (r["status"], r["error"]) == (status, msg), r
    # the largest fine-stage angle count the angular covariance takes: 6144 doubles = 48 KB
    (r,) = plan([plan_request(CFG2, 1081, 8, window(side, 0.05, angle_offset=3071.5 * 0.001, angle_res=0.001, fine=1))])
    assert r["status"] == OK and r["na"] == 6144 and r["need_plain_lut"]


def random_requests(seed=20261015, count=600):
    rng = np.random.default_rng(seed)
    reqs = []
    for _ in range(count):
        res = float(rng.choice([0.01, 0.02, 0.025, 0.03, 0.04, 0.05, 0.08, 0.1]))
        side = int(rng.integers(5, 160))
        p = params((side - 1) * res, res, float(rng.uniform(0.5, 10.0)) * res, float(rng.uniform(1.0, 60.0)))
        mult = float(rng.choice([1, 1, 2, 2, 1.5, 3]))
        if rng.random() < 0.3:
            search = coarse(side, res)
        else:
            half = 0.5 * (int(rng.integers(1, side + 1)) - 1) * res
            search = (half, half, mult * res, mult * res, float(rng.uniform(0.0, 0.6)),
                      float(rng.choice([0.25, 0.5, 1.0, 2.0])) * D, int(rng.random() < 0.2))
        kw = dict(force=int(rng.choice([0, 0, 0, 1, 2, 3])), sat_valid=int(rng.random() < 0.8),
                  high_bytes=int(rng.random() < 0.05))
        if rng.random() < 0.2:  # an angle subset of a split sweep, sometimes empty
            na_full = int(2 * round(search[4] / search[5]) + 1)
            k_first = int(rng.integers(0, na_full + 1))
            kw.update(k_first=k_first, na_override=int(rng.integers(0, na_full - k_first + 1)))
        n = int(rng.choice([1, 90, 360, 720, 1081, 2000, 4000, 7000, 7900, 9000]))
        reqs.append(plan_request(p, n, int(rng.integers(1, 2049)), search, **kw))
    return reqs


def uncovered_rows(r):
    """Origin rows whose lanes touch a grid row that the image of their band does not hold, or that the kernel's band
    clamp moves.  As k_offsets_sorted assigns it, an origin in row y goes to band clamp(floor(y' / band_rows) +
    neg_bands, 0, nbands - 1), y' = y (0 for y < 0 when there are no bands below the grid); as k_sweep_window stages
    it, the unit (band, row tile ty) holds grid rows [(band - neg_bands) * band_rows + stride * 32 * ty, + band_rows +
    halo_rows), and lane l of that tile touches rows y + stride * (32 * ty + l) and the next (its 36 bytes may wrap)."""
    s, br, neg, nb, halo = max(r["stride"], 1), r["band_rows"], r["neg_bands"], r["nbands"], r["halo_rows"]
    H, ty = r["height"], np.arange(r["tiles_y"])
    y = np.arange(-(s * (r["rows_total"] - 1) + 1) - 2 * br, H + 2 * br)
    ye = np.where((y >= 0) | (neg > 0), y, 0)
    raw = ye // br + neg
    band = np.clip(raw, 0, nb - 1)
    lanes = s * (32 * ty[:, None] + np.arange(32)[None, :])  # [ty][lane]
    rows = y[:, None, None, None] + lanes[None, :, :, None] + np.arange(2)[None, None, None, :]
    row0 = (band - neg)[:, None] * br + s * 32 * ty[None, :]
    lo, hi = np.maximum(row0, 0), np.minimum(row0 + br + halo, H)
    in_grid = (rows >= 0) & (rows < H)
    held = (rows >= lo[:, :, None, None]) & (rows < hi[:, :, None, None])
    reaches = in_grid.any(axis=(1, 2, 3))
    bad = (in_grid & ~held).any(axis=(1, 2, 3)) | (reaches & ((raw < 0) | (raw >= nb)))
    return y[bad]


def test_invariants_over_random_geometries(plan):
    out = plan(random_requests())
    kinds = {"window": 0, "banded": 0, "generic": 0, "refused": 0}
    for r in out:
        if r["status"] != OK:
            kinds["refused"] += 1
            continue
        if not r["use_window"]:
            kinds["generic"] += 1
            assert r["need_plain_lut"]
            continue
        kinds["banded" if r["nbands"] > 1 else "window"] += 1
        assert r["stride"] in (1, 2) and r["width_step"] % 8 == 0, r
        # the image, its guards and the kernel's static shared memory fit the opt-in limit
        assert r["win_smem"] + WIN_STATIC <= OPTIN, r
        assert r["osm"] <= LIST_SMEM_MAX, r
        if r["nbands"] == 1:
            assert r["win_smem"] >= r["copy_bytes"] + 2 * 128, r
            continue
        assert r["band_rows"] % 2 == 0 and r["band_rows"] >= 8 and r["nbands"] <= WIN_MAX_BANDS, r
        assert r["band_bytes"] == (r["band_rows"] + r["halo_rows"]) * r["width_step"], r
        assert len(uncovered_rows(r)) == 0, (r, uncovered_rows(r)[:8])
    assert min(kinds.values()) >= 20, kinds
