"""CPU: the oracle of the orientation / command stages (oracle/command_oracle.cpp) against the reference's own compiled code
(oracle/_ref/libref_command.so: Utils::quat_to_euler and MovingWindowFilter, where that build exists) and against the committed fixture
tests/golden/command_v1.npz (tests/golden/make_command_golden.py), bit for bit."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from command_scenarios import DT, HEIGHT0, HMAX, HMIN, KP_LINEAR, KP_LOCK, VARIANTS, quat_from_euler  # noqa: E402
from oracle import command_oracle_py as CO  # noqa: E402
from oracle import ref_command_py as RC  # noqa: E402

needs_ref = pytest.mark.skipif(not RC.available(), reason="oracle/_ref/libref_command.so not built (reference sources absent)")


@pytest.fixture(scope="module")
def G():
    with np.load(os.path.join(ROOT, "tests", "golden", "command_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _quats(n, seed):
    """random non-unit quaternions (|q| - 1 up to 1e-3), and near-gimbal ones with 2 (w y - z x) on both sides of +-1"""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((4, n))
    q /= np.linalg.norm(q, axis=0)
    q *= 1.0 + rng.uniform(-1e-3, 1e-3, n)
    p = np.sign(rng.standard_normal(n)) * (np.pi / 2 - np.abs(rng.normal(0, 1e-6, n)))
    g = quat_from_euler(rng.uniform(-np.pi, np.pi, n), p, rng.uniform(-np.pi, np.pi, n)) * (1.0 + rng.uniform(-1e-3, 1e-3, n))
    return np.concatenate([q, g, np.array([[0.7071067811865476, 0.0, 0.7071067811865476 * (1 + 1e-3), 0.0]]).T], axis=1)


@needs_ref
def test_quat_to_euler_matches_reference_bits():
    q = _quats(20000, 1)
    t2 = 2 * (q[0] * q[2] - q[3] * q[1])
    assert (np.abs(t2) >= 1).sum() > 100 and (np.abs(t2) < 1).sum() > 100
    assert np.array_equal(CO.quat_to_euler(q), RC.quat_to_euler(q))


@needs_ref
def test_moving_window_matches_reference_bits():
    rng = np.random.default_rng(2)
    for W in (1, 2, 5, 60, 100):
        for x in (rng.standard_normal(400), 1e9 + rng.standard_normal(400), np.concatenate([1e16 * np.ones(20), rng.standard_normal(80)])):
            assert np.array_equal(CO.window(W, x), RC.window(W, x)), W


@needs_ref
def test_fixture_pins_are_the_reference(G):
    V, T = G["quat"].shape[:2]
    for v in range(V):
        for t in range(T):
            assert np.array_equal(RC.quat_to_euler(G["quat"][v, t]), G["euler"][v, t])
    for x, y in zip(G["win_x"], G["win_y"]):
        assert np.array_equal(RC.window(5, x), y)


def test_oracle_replays_fixture(G):
    """the oracle's whole orientation + command chain, terrain overrides of root_euler_d[1] in between, against the fixture"""
    V, T, _, R = G["quat"].shape
    assert V == len(VARIANTS)
    for x, y in zip(G["win_x"], G["win_y"]):
        assert np.array_equal(CO.window(5, x), y)
    for v in VARIANTS:
        ori = CO.Orientation(R, filtered=(v != 1))
        com = CO.Command(R, v, HEIGHT0[v], HMIN, HMAX, KP_LINEAR, KP_LOCK)
        row1 = np.zeros(R)
        for t in range(T):
            o = ori(G["quat"][v, t], G["gyro"][v, t], G["acc"][v, t])
            for k in ("rot", "rot_z", "euler", "ang_vel", "imu_acc", "imu_ang_vel"):
                assert np.array_equal(o[k], G[k][v, t]), (v, t, k)
            ov = G["pitch_override"][v, t]
            row1 = np.where(np.isnan(ov), row1, ov)
            mode, kp, ref, des = com(DT, G["cmd"][v, t], G["root_pos"][v, t], row1)
            row1 = ref[1].copy()
            for k, got in zip(("movement_mode", "kp_linear", "ref", "des"), (mode, kp, ref, des)):
                assert np.array_equal(got, G[k][v, t]), (v, t, k)


def test_fixture_covers_the_cases(G):
    """toggles both ways, both sides of the 0.05 velocity threshold, both height clamps, yaw across +-pi, |t2| >= 1, all variants"""
    mm = G["movement_mode"].astype(int)
    assert ((np.diff(mm, axis=1) == 1).any() and (np.diff(mm, axis=1) == -1).any())
    v = np.hypot(G["cmd"][:, :, 0], G["cmd"][:, :, 1])
    walking = mm == 1
    assert (v[walking] > 0.05).any() and (v[walking] < 0.05).any() and np.abs(v - 0.05).min() > 1e-9
    h = G["des"][:, :, 5]
    assert (h == HMIN).any() and (h == HMAX).any()
    yaw = G["euler"][:, :, 2]
    assert (np.abs(np.diff(yaw, axis=1)) > np.pi).any()
    q = G["quat"]
    assert (np.abs(2 * (q[:, :, 0] * q[:, :, 2] - q[:, :, 3] * q[:, :, 1])) >= 1).any()
    # the hardware variant assigns the rates, the others integrate them
    assert np.array_equal(G["ref"][1, :, 0], G["cmd"][1, :, 3]) and not np.array_equal(G["ref"][0, :, 0], G["cmd"][0, :, 3])
    # only Gazebo sets root_lin_vel_d[2] = velz (GazeboA1ROS.cpp:152); hardware and Isaac leave it at 0 (HardwareA1ROS.cpp:121-123,
    # IsaacA1ROS.cpp:99-101) although their joystick commands velz for the height: ref row 7 and des row 8
    velz = G["cmd"][:, :, 2]
    assert (velz[1] != 0).any() and (velz[2] != 0).any()
    assert np.array_equal(G["ref"][0, :, 7], velz[0]) and np.array_equal(G["des"][0, :, 8], velz[0])
    for v in (1, 2):
        assert (G["ref"][v, :, 7] == 0.0).all() and (G["des"][v, :, 8] == 0.0).all(), v
