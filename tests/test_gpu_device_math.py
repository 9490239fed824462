"""The nvcc DEVICE build of the library's shared math headers against their host build, the C library and mpmath,
function by function (tests/device_math_check.cu, built with the library's NVCC_FLAGS).  Hector exact mode, the de-skew
node and the PL-ICP / Karto tolerances rest on these functions; the whole-kernel tests only sample recorded streams.

- glibc_sincosf, both glibc builds (FMA and separate multiply / add): every 61st float with |x| < 120, every float within
  2^16 ulps of each multiple of pi/2, the build probes +-1024 ulps, the reduction thresholds and the special values.
  Bit-identical to the host restatement below 120, and to the C library for the host's own build.
- hector_trig_exact: (float) of the device's double sin / cos for EVERY float with |a| <= 16, against the C library.
- hector_prob_exact: log_odds_prob for EVERY float in [-128, 64], against the C library's exp.
- ros_math_arith / common_helpers: bit-identical to the host build on ros_math_check's seeded sweep and on crafted
  edges (half-integer ties, +-0, NaN, the int32 / int64 range edges, +-1e6 rad, half-cell boundaries).
- ros_math_libm and sensor_pose_of: device and host each within device_math_reference's bounds of mpmath.

The exhaustive groups compare about 2.2e9 inputs each on the host's threads."""
import os

import pytest

import device_math_reference as ref
from test_device_math_host import build_checker, run_checker

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def groups(tmp_path_factory):
    d = tmp_path_factory.mktemp("device_math")
    return run_checker(build_checker(d), d), d


@pytest.mark.parametrize("build", ["fma", "plain"])
def test_glibc_sincosf_device_equals_host(groups, build):
    g = groups[0]["glibc_sincosf_" + build]
    assert g["inputs_below_120"] > 50_000_000, g
    assert g["mismatches"] == 0, g
    if g["libm_compared"]:
        assert g["libm_mismatches"] == 0, g
    assert g["inputs_above_120"] > 0 and g["nan_not_nan"] == 0, g


def test_hector_trig_exact_every_float(groups):
    g = groups[0]["hector_trig_exact"]
    assert g["inputs"] == 2 * (0x41800000 + 1), g
    assert g["mismatches"] == 0 and g["separate_sin_cos_differ"] == 0, g


def test_hector_prob_exact_every_float(groups):
    g = groups[0]["hector_prob_exact"]
    assert g["inputs"] == 0x42800000 + 1 + 0x43000000 + 1, g
    assert g["mismatches"] == 0, g


def test_ros_math_arith_bit_identical(groups):
    g = groups[0]["ros_math_arith"]
    assert g["inputs"] > 100_000 and g["mismatches"] == 0, g
    for b in ("get_rotation_trace", "get_rotation_i0", "get_rotation_i1", "get_rotation_i2", "time_diff_nsec_negative",
              "time_diff_sec_wraps", "from_sec_rollover", "from_sec_negative"):
        assert g["branches"].get(b, 0) > 0, b


def test_common_helpers_bit_identical(groups):
    g = groups[0]["common_helpers"]
    assert g["mismatches"] == 0 and g["kround_vs_math_h"] == 0, g
    assert all(n > 0 for n in g["ops"].values()), g


def test_ros_math_libm_within_bounds_of_mpmath(groups):
    g, d = groups
    assert g["ros_math_libm"]["inputs"] > 100_000
    m = ref.measure(os.path.join(str(d), "libm_records.bin"))
    print({k: (v["device_max"], v["host_max"]) for k, v in m.items()})
    for name, st in m.items():
        assert st["device_max"] <= ref.BOUND[name], (name, st)
        assert st["host_max"] <= ref.BOUND[name], (name, st)
        assert st["heading_max"] == 0.0, (name, st)
