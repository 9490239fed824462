"""The Hector fleet handles without a GPU: b2s_hector_slam_create_fleet and b2s_hector_node_create_fleet refuse every
bad processor spec, laser and node count before any device is touched, naming the processor or node, and the ctypes
mirror of b2s_hector_map_spec matches the header's layout as a C compiler lays it out."""
import ctypes as C
import importlib
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "creating-2d-laser-slam-from-scratch_b200"
H = importlib.import_module(PKG + ".hector")
N = importlib.import_module(PKG + ".hector_node")
R = importlib.import_module(PKG + ".rosio")
OK, BAD, TOO_LARGE, NO_DEVICE = 0, 1, 7, 5


def _slam_fleet(specs, max_points=1081):
    L = H._bind()
    h = C.c_void_p()
    arr = (H.HectorMapSpec * len(specs))(*specs)
    st = L.b2s_hector_slam_create_fleet(len(specs), max_points, arr, 0, None, C.byref(h))
    return st, h, L.b2s_last_error()


def _geom(n=1081, inc=0.004363323):
    return R.make_msg(-2.356, -2.356 + inc * max(n - 1, 0), inc, 0.1, 30.0, np.zeros(max(n, 0), np.float32))


def _node_fleet(params, geoms, mounts=None):
    L = N._bind()
    h = C.c_void_p()
    B = len(params)
    m = np.ascontiguousarray(mounts if mounts is not None else [(0, 0, 0, 0, 0, 0, 1)] * B, np.float64)
    st = L.b2s_hector_node_create_fleet(B, (N.HectorNodeParams * B)(*params), (R.LaserScanMsg * B)(*geoms),
                                        m.ctypes.data_as(C.POINTER(C.c_double)), 0, C.byref(h))
    return st, h, L.b2s_last_error()


def test_status_codes_are_the_headers(pkg):
    assert (pkg.abi.B2S_ERR_BAD_PARAMS, pkg.abi.B2S_ERR_TOO_LARGE, pkg.abi.B2S_ERR_NO_DEVICE) == (BAD, TOO_LARGE, NO_DEVICE)


@pytest.mark.parametrize("bad, why", [
    (dict(levels=0), b"levels"), (dict(levels=9), b"levels"), (dict(resolution=0.0), b"map_resolution"),
    (dict(resolution=-0.05), b"map_resolution"), (dict(size_x=8, levels=3), b"2 cells"),
    (dict(size_y=11, levels=3), b"2 cells"), (dict(size_x=2, size_y=256, levels=1), b"2 cells"),
])
def test_slam_fleet_refuses_a_bad_spec_naming_the_processor(pkg, bad, why):
    good = [H.map_spec(size_x=512, size_y=512), H.map_spec(resolution=0.025, size_x=1024, size_y=768, levels=4),
            H.map_spec(resolution=0.1, size_x=256, size_y=256, levels=1)]
    for k in range(3):
        specs = list(good)
        specs[k] = H.map_spec(**dict(dict(resolution=0.05, size_x=512, size_y=512, levels=3), **bad))
        st, h, msg = _slam_fleet(specs)
        assert st == BAD and not h.value, (k, bad)
        assert b"processor %d" % k in msg and why in msg, msg


def test_slam_fleet_refuses_counts(pkg):
    spec = H.map_spec(size_x=256, size_y=256)
    assert _slam_fleet([spec], max_points=4097)[0] == TOO_LARGE
    assert _slam_fleet([spec], max_points=0)[0] == BAD
    L = H._bind()
    h = C.c_void_p()
    assert L.b2s_hector_slam_create_fleet(0, 16, (H.HectorMapSpec * 1)(spec), 0, None, C.byref(h)) == BAD
    assert L.b2s_hector_slam_create_fleet(1, 16, None, 0, None, C.byref(h)) == BAD
    assert L.b2s_hector_slam_create_fleet(1, 16, (H.HectorMapSpec * 1)(spec), 0, None, None) == BAD


def _params(**kw):
    return N.node_params(dict(dict(map_size=512), **kw))


@pytest.mark.parametrize("bad, geom_kw, code, why", [
    (dict(map_multi_res_levels=9), {}, BAD, b"levels"),
    (dict(map_size=8, map_multi_res_levels=3), {}, BAD, b"2 cells"),
    (dict(map_size=11, map_multi_res_levels=3), {}, BAD, b"2 cells"),
    (dict(map_resolution=0.0), {}, BAD, b"map_resolution"),
    (dict(map_size=0), {}, BAD, b"map_size"),
    (dict(map_pub_period=0.0), {}, BAD, b"map_pub_period"),
    ({}, dict(n=4097), TOO_LARGE, b"4096"),
    ({}, dict(inc=0.0), BAD, b"angle_increment"),
])
def test_node_fleet_refuses_a_bad_node_naming_it(pkg, bad, geom_kw, code, why):
    params = [_params(), _params(map_size=1024, map_resolution=0.025, map_multi_res_levels=4),
              _params(map_size=256, map_resolution=0.1, map_multi_res_levels=1)]
    geoms = [_geom(1081), _geom(720, 0.008737), _geom(1440, 0.0043633)]
    for k in range(3):
        p, g = list(params), list(geoms)
        p[k] = _params(**bad)
        if geom_kw:
            g[k] = _geom(**geom_kw)
        st, h, msg = _node_fleet(p, g)
        assert st == code and not h.value, (k, bad, geom_kw)
        assert b"node %d" % k in msg and why in msg, msg


def test_node_fleet_refuses_a_bad_mount_and_counts(pkg):
    st, h, msg = _node_fleet([_params(), _params()], [_geom(), _geom()], [(0, 0, 0, 0, 0, 0, 1), (0, 0, 0, 0, 0, 0, 0)])
    assert st == BAD and b"node 1" in msg and not h.value
    B = 65536
    st, h, _ = _node_fleet([_params()] * B, [_geom(8)] * B)
    assert st == TOO_LARGE and not h.value
    L = N._bind()
    h = C.c_void_p()
    assert L.b2s_hector_node_create_fleet(0, None, None, None, 0, C.byref(h)) == BAD
    assert L.b2s_hector_node_create_fleet(1, (N.HectorNodeParams * 1)(_params()), None, None, 0, C.byref(h)) == BAD


def test_no_device_is_an_error(pkg):
    """Without a GPU valid fleets answer NO_DEVICE and hand out no handle: there is no CPU fallback."""
    if pkg.load("matcher").device_count() > 0:
        pytest.skip("a device is present")
    st, h, _ = _slam_fleet([H.map_spec(size_x=256, size_y=256), H.map_spec(levels=4)])
    assert st == NO_DEVICE and not h.value
    st, h, _ = _node_fleet([_params(), _params(map_size=256, map_multi_res_levels=1)], [_geom(1081), _geom(4096)])
    assert st == NO_DEVICE and not h.value


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "b200slam.h"
#define F(f) printf("\"%s\": %zu, ", #f, offsetof(b2s_hector_map_spec, f))
int main(void) {
  printf("{");
  F(map_resolution); F(map_size_x); F(map_size_y); F(start_x); F(start_y); F(levels); F(update_free);
  F(update_occupied); F(min_dist); F(min_angle); F(reserved);
  printf("\"sizeof\": %zu}\n", sizeof(b2s_hector_map_spec));
  return 0;
}
"""


def test_map_spec_matches_the_header(tmp_path):
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(_LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = json.loads(subprocess.check_output([exe], text=True))
    size = got.pop("sizeof")
    assert [f for f, _ in H.HectorMapSpec._fields_] == list(got)
    for f, off in got.items():
        assert getattr(H.HectorMapSpec, f).offset == off, f
    assert C.sizeof(H.HectorMapSpec) == size == 64


def test_map_spec_defaults_are_the_create_defaults():
    s = H.map_spec()
    assert (s.update_free, s.update_occupied) == (np.float32(0.4), np.float32(0.6))
    assert (s.min_dist, s.min_angle) == (np.float32(0.4), np.float32(0.13))
    assert list(s.reserved) == [0] * 6
