"""csrc/glibc_math.cuh restates glibc's sinf / cosf (double-precision polynomial after a one-multiply reduction) so that
the device takes Rotation2Df's sine / cosine exactly as the reference's CPU build does.  The same header compiles for the
host: this test runs it against THIS machine's C library (every 251st float with |x| < 120, both signs, sinf / cosf /
sincosf; the exhaustive run — stride 1, 2 246 049 792 inputs — gave 0 mismatches for the FMA build and 34 for the
plain one on the build container, glibc 2.39)."""
import json
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_restated_sincosf_equals_host_libm(tmp_path):
    exe = str(tmp_path / "glibc_math_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread",
                           os.path.join(HERE, "glibc_math_check.cpp"), "-o", exe])
    out = json.loads(subprocess.check_output([exe, "251"], text=True))
    assert out["inputs"] > 8_000_000
    assert out["host_variant"] in (0, 1), out
    key = "mismatch_fma" if out["host_variant"] == 1 else "mismatch_plain"
    assert out[key] == 0, out


def test_normalize_angle_shortcut_equals_fmod(tmp_path):
    """util_normalize_angle's |a| < 2 pi path (one add, one compare, one subtract in double) against the two fmod calls of
    util::normalize_angle on this machine's C library: identical bits."""
    exe = str(tmp_path / "normalize_angle_check")
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", os.path.join(HERE, "normalize_angle_check.c"), "-o", exe, "-lm"])
    out = json.loads(subprocess.check_output([exe, "20000000"], text=True))
    assert out["inputs"] > 20_000_000 and out["mismatches"] == 0, out
