"""The lesson3 odometry fleet handle (b2s_plicp_odom_create_fleet) without a GPU: every refusal comes before the
device is touched and names the recording, a valid fleet is refused with NO_DEVICE instead of falling back to the CPU,
and the laser struct's ctypes mirror matches the header as a C compiler lays it out."""
import ctypes as C
import importlib
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
abi = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.abi")
P = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.plicp")
BAD, NO_DEVICE = abi.B2S_ERR_BAD_PARAMS, abi.B2S_ERR_NO_DEVICE


def _laser(n=1081, reserved=0):
    return abi.PlicpOdomLaser(n, -2.35619449, 0.00436332313, reserved)


def _create(batch, params, lasers, out=True):
    L = P._bind()
    h = C.c_void_p()
    pa = (abi.PlicpOdomParams * max(len(params), 1))(*params) if params is not None else None
    la = (abi.PlicpOdomLaser * max(len(lasers), 1))(*lasers) if lasers is not None else None
    st = L.b2s_plicp_odom_create_fleet(batch, pa, la, 0, None, C.byref(h) if out else None)
    return st, h


def _err():
    return importlib.import_module("creating-2d-laser-slam-from-scratch_b200.matcher").lib().b2s_last_error().decode()


@pytest.mark.parametrize("bad, what", [
    (lambda p, l: l.__setattr__("n_beams", 2), "fewer than 3 beams"),
    (lambda p, l: l.__setattr__("n_beams", -1), "fewer than 3 beams"),
    (lambda p, l: l.__setattr__("reserved", 1), "reserved"),
    (lambda p, l: p.icp.__setattr__("max_iterations", 0), "max_iterations"),
    (lambda p, l: [p.base_to_laser.__setitem__(k, 0.0) for k in range(3, 7)], "quaternion"),
    (lambda p, l: p.base_to_laser.__setitem__(6, float("nan")), "quaternion"),
    (lambda p, l: p.base_to_laser.__setitem__(5, float("inf")), "quaternion"),
])
def test_create_refusals_name_the_recording(pkg, bad, what):
    """A bad row of recording 2 of 4 is refused with BAD_PARAMS, on any machine, and the message names recording 2."""
    params = [abi.plicp_odom_params() for _ in range(4)]
    lasers = [_laser(n) for n in (1081, 360, 720, 2408)]
    bad(params[2], lasers[2])
    st, h = _create(4, params, lasers)
    assert st == BAD and not h
    msg = _err()
    assert "recording 2" in msg and what in msg, msg


def test_create_null_and_batch_refusals(pkg):
    params, lasers = [abi.plicp_odom_params()] * 2, [_laser(), _laser(360)]
    for args in ((0, params, lasers), (-1, params, lasers), (2, None, lasers), (2, params, None)):
        assert _create(*args)[0] == BAD
    assert _create(2, params, lasers, out=False)[0] == BAD
    with pytest.raises(pkg.load("matcher").B2SError) as e:
        P.Odometry.fleet([abi.plicp_odom_params()], [2], [-1.0], [0.01])
    assert e.value.status == BAD and "recording 0" in str(e.value)
    with pytest.raises(ValueError):
        P.Odometry.fleet([abi.plicp_odom_params()] * 2, [360], [-1.0], [0.01])


def test_process_refusals_need_no_handle(pkg):
    L = P._bind()
    assert L.b2s_plicp_odom_process_fleet(None, None, None, None, None, None) == BAD
    assert L.b2s_plicp_odom_process(None, None, None, None, None) == BAD


def test_no_device_is_an_error(pkg):
    """Without a GPU a valid fleet answers NO_DEVICE and hands out no handle: there is no CPU fallback."""
    if pkg.load("matcher").device_count() > 0:
        pytest.skip("a device is present")
    st, h = _create(3, [abi.plicp_odom_params()] * 3, [_laser(3), _laser(2408), _laser(5000)])
    assert st == NO_DEVICE and not h
    with pytest.raises(pkg.load("matcher").B2SError) as e:
        P.Odometry.fleet([abi.plicp_odom_params()] * 2, [360, 720], [-3.14, -3.14], [0.0174, 0.0087])
    assert e.value.status == NO_DEVICE


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "b200slam.h"
#define F(T, f) printf("\"%s.%s\": %zu, ", #T, #f, offsetof(T, f))
int main(void) {
  printf("{");
  F(b2s_plicp_odom_laser, n_beams); F(b2s_plicp_odom_laser, angle_min); F(b2s_plicp_odom_laser, angle_increment);
  F(b2s_plicp_odom_laser, reserved);
  printf("\"size\": %zu}\n", sizeof(b2s_plicp_odom_laser));
  return 0;
}
"""


def test_laser_struct_matches_the_header(tmp_path):
    src, exe = tmp_path / "layout.c", str(tmp_path / "layout")
    src.write_text(_LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = json.loads(subprocess.check_output([exe], text=True))
    T = abi.PlicpOdomLaser
    assert [f for f, _ in T._fields_] == [k.split(".", 1)[1] for k in got if k.startswith("b2s_plicp_odom_laser.")]
    for f, _ in T._fields_:
        assert getattr(T, f).offset == got[f"b2s_plicp_odom_laser.{f}"], f
    assert C.sizeof(T) == got["size"] == 16
