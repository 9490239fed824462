"""The lesson5 de-skew node handle (b2s_deskew_node_*) without a GPU: create refuses bad arguments before any device
is touched, refuses to run without a device instead of falling back, and the ctypes structs match the header's
layout as a C compiler lays it out."""
import ctypes as C
import importlib
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DS = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.deskew")
BAD, NO_DEVICE = 1, 5


def _create(batch, lasers, out=True):
    L = DS._bind()
    h = C.c_void_p()
    arr = (DS.DeskewLaser * max(len(lasers), 1))(*lasers) if lasers is not None else None
    return L.b2s_deskew_node_create(batch, arr, 0, None, C.byref(h) if out else None), h


def _laser(n=8):
    return DS.DeskewLaser(-1.0, 0.01, n, 1, 1, 0)


def test_create_refusals_need_no_device(pkg):
    """batch < 1, a laser without beams and NULL pointers are refused before the device is touched, on any machine."""
    assert _create(0, [_laser()])[0] == BAD
    assert _create(-3, [_laser()])[0] == BAD
    assert _create(2, [_laser(), _laser(0)])[0] == BAD
    assert _create(1, [_laser(-5)])[0] == BAD
    assert _create(1, None)[0] == BAD
    assert _create(1, [_laser()], out=False)[0] == BAD
    L = DS._bind()
    assert L.b2s_deskew_node_reset(None, -1) == BAD
    assert L.b2s_deskew_node_process(*([None] * 11)) == BAD
    L.b2s_deskew_node_destroy(None)


def test_no_device_is_an_error(pkg):
    """Without a GPU a valid create answers NO_DEVICE and hands out no handle: there is no CPU fallback."""
    if pkg.load("matcher").device_count() > 0:
        pytest.skip("a device is present")
    st, h = _create(2, [_laser(), _laser(1081)])
    assert st == NO_DEVICE and not h
    with pytest.raises(pkg.load("matcher").B2SError) as e:
        DS.DeskewNodeBatch([_laser()])
    assert e.value.status == NO_DEVICE


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "b200slam.h"
#define F(T, f) printf("\"%s.%s\": %zu, ", #T, #f, offsetof(T, f))
int main(void) {
  printf("{");
  F(b2s_deskew_laser, angle_min); F(b2s_deskew_laser, angle_increment); F(b2s_deskew_laser, n_beams);
  F(b2s_deskew_laser, use_imu); F(b2s_deskew_laser, use_odom); F(b2s_deskew_laser, reserved);
  F(b2s_deskew_node_scan, sec); F(b2s_deskew_node_scan, nsec); F(b2s_deskew_node_scan, time_increment);
  F(b2s_deskew_node_scan, range_min); F(b2s_deskew_node_scan, range_max); F(b2s_deskew_node_scan, imu_arrived);
  F(b2s_deskew_node_scan, odom_arrived); F(b2s_deskew_node_scan, reserved);
  F(b2s_imu_msg, sec); F(b2s_imu_msg, nsec); F(b2s_imu_msg, angular_velocity);
  F(b2s_odom_msg, sec); F(b2s_odom_msg, nsec); F(b2s_odom_msg, position); F(b2s_odom_msg, orientation);
  F(b2s_deskew_scan, time_start); F(b2s_deskew_scan, time_increment); F(b2s_deskew_scan, range_min);
  F(b2s_deskew_scan, range_max); F(b2s_deskew_scan, use_imu); F(b2s_deskew_scan, use_odom); F(b2s_deskew_scan, imu_last);
  F(b2s_deskew_scan, reserved); F(b2s_deskew_scan, odom_start_time); F(b2s_deskew_scan, odom_end_time);
  F(b2s_deskew_scan, odom_incre); F(b2s_deskew_scan, reserved2);
  printf("\"sizes\": [%zu, %zu, %zu, %zu, %zu], \"cached\": %d}\n", sizeof(b2s_deskew_laser), sizeof(b2s_deskew_node_scan),
         sizeof(b2s_imu_msg), sizeof(b2s_odom_msg), sizeof(b2s_deskew_scan), B2S_DESKEW_CACHED);
  return 0;
}
"""


def test_structs_match_the_header(tmp_path):
    """Every field offset and struct size of the ctypes mirrors equals the C compiler's layout of include/b200slam.h,
    and CACHED is the header's B2S_DESKEW_CACHED."""
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(_LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = json.loads(subprocess.check_output([exe], text=True))
    mirrors = {"b2s_deskew_laser": DS.DeskewLaser, "b2s_deskew_node_scan": DS.NodeScan, "b2s_imu_msg": DS.ImuMsg,
               "b2s_odom_msg": DS.OdomMsg, "b2s_deskew_scan": DS.DeskewScan}
    for name, T in mirrors.items():
        fields = [f for f, _ in T._fields_]
        assert fields == [k.split(".", 1)[1] for k in got if k.startswith(name + ".")], name
        for f in fields:
            assert getattr(T, f).offset == got[f"{name}.{f}"], (name, f)
    assert [C.sizeof(T) for T in mirrors.values()] == got["sizes"]
    assert got["cached"] == DS.CACHED == 7
