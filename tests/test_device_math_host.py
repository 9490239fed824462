"""The CPU half of tests/device_math_check.cu (see tests/test_gpu_device_math.py): the checker compiles with nvcc and the
library's own flags, and its host half runs without a GPU.  glibc_math.cuh's host restatement of BOTH glibc sinf / cosf
builds against this machine's C library on every 61st float with |x| < 120; kround against Math.h's form; and the host
C library's values of the ros_math.cuh / common.cuh functions that call libm against mpmath, within the bounds of
device_math_reference."""
import importlib
import json
import os
import subprocess

import pytest

import device_math_reference as ref

HERE = os.path.dirname(os.path.abspath(__file__))


def build_checker(out_dir, flags=None):
    """nvcc device_math_check.cu with the library's NVCC_FLAGS (or `flags`), host side without FP contraction, libm"""
    build = importlib.import_module("creating-2d-laser-slam-from-scratch_b200.build")
    exe = os.path.join(str(out_dir), "device_math_check")
    subprocess.check_call([build.nvcc()] + list(flags or build.NVCC_FLAGS) +
                          ["-Xcompiler", "-ffp-contract=off", os.path.join(HERE, "device_math_check.cu"), "-o", exe, "-lm"])
    return exe


def run_checker(exe, out_dir, *args):
    """-> {group: its JSON line}"""
    out = subprocess.run([exe, "--out", str(out_dir)] + list(args), capture_output=True, text=True, check=True).stdout
    return {g["group"]: g for g in map(json.loads, out.splitlines())}


@pytest.fixture(scope="module")
def host_half(tmp_path_factory):
    d = tmp_path_factory.mktemp("device_math_host")
    return run_checker(build_checker(d), d, "--host-only"), d


def test_both_glibc_builds_restated_on_host(host_half):
    g, _ = host_half
    variant = g["setup"]["host_variant"]
    assert variant in (0, 1), g["setup"]
    for name, v in (("host_glibc_sincosf_fma", 1), ("host_glibc_sincosf_plain", 0)):
        assert g[name]["inputs"] > 36_000_000, g[name]
        if v == variant:
            assert g[name]["libm_mismatches"] == 0, g[name]
        else:  # the other build differs from this libm on 34 floats of the whole range, next to multiples of pi/2
            assert g[name]["libm_mismatches"] <= 34, g[name]


def test_kround_is_math_h_round(host_half):
    g, _ = host_half
    c = g["common_helpers"]
    assert c["ops"]["kround"] > 500 and c["kround_vs_math_h"] == 0, c


def test_host_libm_values_against_mpmath(host_half):
    g, d = host_half
    assert g["ros_math_libm"]["inputs"] > 100_000, g["ros_math_libm"]
    for b in ("get_rpy", "get_rpy_singular_up", "get_rpy_singular_down", "tf2_yaw", "tf2_yaw_sarg_low",
              "tf2_yaw_sarg_high"):
        assert g["ros_math_libm"]["branches"].get(b, 0) > 0, b
    m = ref.measure(os.path.join(str(d), "libm_records.bin"), with_device=False)
    assert set(m) == set(ref.BOUND), m
    for name, st in m.items():
        assert st["host_max"] <= ref.BOUND[name], (name, st)
        assert st["heading_max"] == 0.0, (name, st)
