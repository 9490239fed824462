"""lesson3's PL-ICP odometry node (ScanMatchPLICP, plicp_odometry.cc:191-517) restated in C (orc_plicp_odometry) against
the unmodified node and an independent float64 statement of its tf chain (CPU).

The node is compiled where it lies against ROS, tf2 and CSM stand-ins (oracle/ref_lesson3.cpp), its sm_icp answered by
the PL-ICP restatement, live where oracle/_ref/ is built and from tests/golden/reference/ elsewhere.  Every line of the
node that runs is pinned; sm_icp (CSM) and tf2's LinearMath are restated, so they are not."""
import math

import numpy as np
import pytest

import plicp_odometry_cases as pc
from oracle import ref_lesson3


@pytest.fixture(scope="module")
def answers():
    return pc.node_answers(ref_lesson3.available())


@pytest.fixture(scope="module")
def restated():
    return {name: pc.restate(st) for name, st in pc.STREAMS.items()}


@pytest.mark.parametrize("name", sorted(pc.STREAMS))
def test_restatement_equals_node(answers, restated, name):
    """Every published pose, quaternion, twist, first guess, sm_icp result and key-frame decision, bit for bit."""
    mine, node = pc.pack(restated[name]), answers[name]
    same = (mine.view(np.int64) == node.view(np.int64)) | (np.isnan(mine) & np.isnan(node))
    assert same.all(), f"{name}: scan / column {np.argwhere(~same)[0].tolist()} differ from the node"


def test_streams_cover_the_node(restated):
    """Each stream produces the event it is named for."""
    S = restated
    d5 = math.radians(5.0)

    def kf_by(name, rule):
        return [k for k, s in enumerate(S[name]) if s["published"] and s["keyframe"] and rule(s)]

    assert (S["straight"]["first_guess"][2:, 0] != 0).all(), "no constant-velocity prediction"
    assert kf_by("rotation", lambda s: abs(s["angular"][2] * 0.1) > d5), "no key frame by rotation"
    back = S["backward"][2:]
    assert (back["linear"][:, 0] < 0).all(), "backward drive left a velocity that predicts"
    stop = S["stop_and_go"]
    assert any(s["valid"] and s["x"][0] == 0 and s["x"][1] == 0 for s in stop), "no exact zero motion"
    assert kf_by("scan_count", lambda s: True) and all(
        math.hypot(*s["x"][:2]) < 0.1 for s in S["scan_count"][1:]), "scan-count rule did not fire alone"
    for name in ("launch_mount", "yaw_pi_mount"):
        assert pc.STREAMS[name]["mount"][2] == 0.254
    assert np.any(np.diff(pc.STREAMS["jitter_stamps"]["stamps"][:, 0]) > 0) and \
        np.any(pc.STREAMS["jitter_stamps"]["stamps"][:, 1] > 900_000_000), "jitter does not cross a second"
    eq = S["equal_stamps"]
    assert np.isinf(eq["linear"][18, 0]), "equal stamps did not give dt = 0"
    nv = S["no_valid_reading"]
    assert not nv["valid"][6] and not nv["valid"][14], "an empty scan matched"
    assert pc.STREAMS["params"]["params"]["kf_scan_count"] == 4 and kf_by("params", lambda s: True)


def _h(x, y, yaw):
    c, s = math.cos(yaw), math.sin(yaw)
    return np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0], [0, 0, 0, 1.0]])


def _mount(m):
    x, y, z, w = m[3:]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R / (x * x + y * y + z * z + w * w), m[:3]
    return T


@pytest.mark.parametrize("name", sorted(pc.STREAMS))
def test_float64_chain(restated, name):
    """A numpy statement of the node's chain with 4x4 homogeneous matrices, driven by the restatement's own sm_icp
    results, rebuilds every published pose and every first guess to 1e-12."""
    st, out = pc.STREAMS[name], restated[name]
    b2l = _mount(st["mount"])
    l2b = np.linalg.inv(b2l)
    bio, kf, vx, last = np.eye(4), np.eye(4), 0.0, None
    for k, s in enumerate(out):
        t = int(st["stamps"][k][0]) + 1e-9 * int(st["stamps"][k][1])
        if k == 0:
            last = t
            continue
        dt = t - last
        with np.errstate(invalid="ignore", over="ignore"):
            pred = _h(0.0 if vx < 1e-6 else dt * vx, 0.0, 0.0) @ (bio @ np.linalg.inv(kf))
            pl = l2b @ np.linalg.inv(bio) @ pred @ bio @ b2l
        if np.all(np.isfinite(pl)):
            g = (pl[0, 3], pl[1, 3], math.atan2(pl[1, 0], pl[0, 0]))
            assert np.allclose(s["first_guess"], g, rtol=0, atol=1e-12), (k, s["first_guess"], g)
        corr = np.eye(4)
        if s["valid"]:
            corr = b2l @ _h(*s["x"]) @ l2b
            bio = kf @ corr
            with np.errstate(divide="ignore", invalid="ignore"):
                vx = corr[0, 3] / dt if abs(dt) > 0 else s["linear"][0]
        assert np.allclose(s["position"][:2], bio[:2, 3], rtol=0, atol=1e-12)
        yaw = math.atan2(bio[1, 0], bio[0, 0])
        q = s["orientation"]
        assert abs(math.remainder(2 * math.atan2(q[2], q[3]) - yaw, 2 * math.pi)) < 1e-12
        if s["keyframe"]:
            kf = bio.copy()
        last = t


def test_noise_free_trajectory_recovered():
    """On a noise-free synthetic drive (3 cm and 0.5 deg per scan) the published poses follow the true base poses to
    5 mm and 0.1 deg after 40 scans: each key-frame match is exact up to the matcher's convergence (epsilon 1e-6 per
    iteration, at most 10 iterations) and the beam discretisation of the point-to-line fit, and the error of key-frame
    links adds up over the ~10 links of the run."""
    st = pc.stream(21, [(0.03, 0.0, math.radians(0.5))] * 40, sigma=0.0)
    out = pc.restate(st)
    p0 = st["poses"][0]
    for k in range(1, len(out)):
        c, s = math.cos(-p0[2]), math.sin(-p0[2])
        dx, dy = st["poses"][k][:2] - p0[:2]
        true = (c * dx - s * dy, s * dx + c * dy, st["poses"][k][2] - p0[2])
        q = out[k]["orientation"]
        yaw = 2 * math.atan2(q[2], q[3])
        assert math.hypot(out[k]["position"][0] - true[0], out[k]["position"][1] - true[1]) < 5e-3, k
        assert abs(math.remainder(yaw - true[2], 2 * math.pi)) < math.radians(0.1), k


def test_create_without_device(pkg):
    """No CPU fallback: without a device create is refused with NO_DEVICE; bad arguments are refused first."""
    P = pkg.load("plicp")
    M = pkg.load("matcher")
    abi = pkg.abi
    with pytest.raises(M.B2SError) as e:
        P.Odometry(abi.plicp_odom_params(), 0, 1081, *map(float, pc.FIELDS))
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    with pytest.raises(M.B2SError) as e:
        P.Odometry(abi.plicp_odom_params(base_to_laser=(0, 0, 0, 0, 0, 0, 0)), 1, 1081, *map(float, pc.FIELDS))
    assert e.value.status == abi.B2S_ERR_BAD_PARAMS
    if M.device_count() > 0:
        return
    with pytest.raises(M.B2SError) as e:
        P.Odometry(abi.plicp_odom_params(), 4, 1081, *map(float, pc.FIELDS))
    assert e.value.status == abi.B2S_ERR_NO_DEVICE
