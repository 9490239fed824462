"""tf / tf2 LinearMath and roscpp Time / Duration are defined three times: in the library (csrc/ros_math.cuh, host and
device), in the C restatements (oracle/linear_math.h) and in the stand-ins the unmodified nodes build against
(oracle/shim/tf2, oracle/shim/tf, oracle/shim_lesson6/tf/tf_core.h, oracle/shim/ros/ros.h).  tf and roscpp are not in
the reference tree, so no node recording pins this arithmetic; this test holds the three equal bit for bit on a seeded
sweep that reaches the branches node streams rarely take: getRotation with trace <= 0 (i = 0, 1, 2), getRPY at
|m[2][0]| >= 1, tf2::getYaw at |sarg| >= 0.99999, negative nanosecond differences, the int32 wrap of seconds and the
fromSec rollover."""
import json
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE = os.path.join(os.path.dirname(HERE), "oracle")

BRANCHES = ["get_rotation_trace", "get_rotation_i0", "get_rotation_i1", "get_rotation_i2", "get_rpy",
            "get_rpy_singular_up", "get_rpy_singular_down", "tf2_yaw", "tf2_yaw_sarg_low", "tf2_yaw_sarg_high",
            "time_diff_nsec_negative", "time_diff_nsec_positive", "time_diff_sec_wraps", "from_sec_rollover",
            "from_sec_negative"]


def test_library_restatements_and_stand_ins_agree(tmp_path):
    exe = str(tmp_path / "ros_math_check")
    # -fwrapv: roscpp's Time - Time subtracts the seconds as int32, which wraps across 2^31 (signed overflow otherwise)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fwrapv",
                           "-I" + os.path.join(ORACLE, "shim"), "-I" + os.path.join(ORACLE, "shim_lesson6"),
                           os.path.join(HERE, "ros_math_check.cpp"), "-o", exe])
    out = json.loads(subprocess.check_output([exe], text=True))
    assert out["mismatches"] == 0, out
    assert out["checks"] > 1_000_000, out
    for b in BRANCHES:
        assert out["branches"].get(b, 0) > 0, (b, out["branches"])
