"""The staged layouts of the angle-pruning bound's 4x4 and 7x7 pooled images (csrc/karto_sweep_plan.cuh pool_layout:
four planes split by the residue of f + lead modulo 4, each with zero padding), checked without a GPU by
tests/pool_layout_check.cu on seeded grids: every P[f] has its own byte in its own plane and the padding is zero, and,
for the 4x4 image of the single-angle pass, every interior beam's block-row read stays in its plane and keeps exactly
the pooled values at its 8 block corners.  Geometries: the benchmark's (width_step 408), the range
thresholds that give the other width_step classes modulo 32 (384, 392, 400), a small grid (width_step 48) whose
interior windows reach both ends of the data, a wider one (width_step 488), and a 24 x 24 grid whose few interior
windows have corners past the last byte of the data, read from the planes' padding."""
import importlib
import json
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GEOMS = {408: (1.5, 0.05, 0.03, 9.25), 384: (1.5, 0.05, 0.03, 8.6), 392: (1.5, 0.05, 0.03, 8.8),
         400: (1.5, 0.05, 0.03, 8.95), 48: (1.5, 0.05, 0.03, 0.3), 488: (1.5, 0.05, 0.03, 11.2),
         24: (0.55, 0.05, 0.03, 0.2)}


@pytest.fixture(scope="module")
def layout(tmp_path_factory):
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    exe = str(tmp_path_factory.mktemp("pool_layout") / "pool_layout_check")
    subprocess.check_call([build.nvcc(), "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a",
                           os.path.join(HERE, "pool_layout_check.cu"), "-o", exe])

    def run(geom, seed, K=4):
        req = " ".join(repr(v) for v in (*geom, seed, K)) + "\n"
        out = subprocess.run([exe], input=req, capture_output=True, text=True, check=True)
        return json.loads(out.stdout)

    return run


@pytest.mark.parametrize("ws", sorted(GEOMS))
def test_planes_hold_every_pooled_value_and_every_interior_read(layout, ws):
    r = layout(GEOMS[ws], seed=ws)
    assert r["width_step"] == ws and r["ok"], r
    assert r["interior"] > 0
    # a plane is (pool_lead + data_size) / 4 bytes of P and at least 32 of zeros, 16-byte aligned; the reads stay in it
    assert r["plane"] % 16 == 0 and r["plane"] >= (4 * ws + r["data_size"]) // 4 + 32, r
    assert r["pool_bytes"] == 4 * r["plane"] and r["max_read_end"] <= r["plane"], r
    if ws == 24:
        assert r["max_read_end"] > (4 * ws + r["data_size"]) // 4 + 8, r  # corners in the padding, not only the read


@pytest.mark.parametrize("ws", sorted(GEOMS))
def test_7x7_planes_hold_every_pooled_value(layout, ws):
    """the group pass's image: a lead of 8 rows, the same planes, padding and pitch rules"""
    r = layout(GEOMS[ws], seed=ws, K=7)
    assert r["width_step"] == ws and r["ok"], r
    assert r["lead"] == 8 * ws and r["interior"] == 0, r
    assert r["plane"] % 16 == 0 and r["plane"] >= (8 * ws + r["data_size"]) // 4 + 32, r
    assert r["pool_bytes"] == 4 * r["plane"] and r["pitch"] % 128 == 0 and r["pitch"] >= r["pool_bytes"], r
