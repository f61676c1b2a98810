"""CPU: the unchanged device code of a1mpc_swing.cuh (swing_legs_kernel, terrain_pitch_kernel) on the block emulator against the oracle's
restatement, tick by tick, with the tolerances of the GPU suite."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_swing_py as E  # noqa: E402
from oracle import swing_oracle_py as SO  # noqa: E402
from swing_scenarios import CPS, KD_RESET, KD_ROS, KP_RESET, KP_ROS, Scenario, check_tick  # noqa: E402

DT = 0.0025


def run(B, T, seed, kp, kd, adapt):
    sc = Scenario(B, seed)
    state = E.swing_init(B)
    ora = SO.Swing(B)
    worst = [0.0, 0.0]
    seen = dict(early=False, neg=False, pos=False)
    for t in range(T):
        x = sc.tick()
        args = (x["gait_counter"], x["plan_contacts"], x["rot_z"], x["foot_pos_abs"], x["foot_pos_target_rel"], x["foot_force"])
        fk, con, cur, rc = E.swing_legs(state, CPS, DT, kp, kd, *args)
        fk0, con0, cur0, rc0 = ora.legs(CPS, DT, kp, kd, *args)
        ref, ref0 = np.full((9, B), 3.0), np.full((9, B), 3.0)
        pitch = E.terrain_pitch(state, adapt, x["root_pos"], ref)
        pitch0 = ora.terrain(adapt, x["root_pos"], ref0)
        ef, ea = check_tick((fk, con, rc, pitch, ref[1]), (fk0, con0, rc0, pitch0, ref0[1]), "tick %d" % t)
        assert np.array_equal(np.delete(ref, 1, axis=0), np.full((8, B), 3.0))
        assert np.abs(cur - cur0).max() <= 1e-15
        worst = [max(worst[0], ef), max(worst[1], ea)]
        seen["early"] |= bool(((con & ~x["plan_contacts"]) != 0).any())
        seen["neg"] |= bool((ref[1] == -0.5).any())
        seen["pos"] |= bool((ref[1] == 0.5).any())
    return worst, seen


def test_emulated_kernels_match_the_oracle_256_robots_300_ticks():
    worst, seen = run(256, 300, 31, KP_RESET, KD_RESET, 1)
    assert all(seen.values()), seen


def test_emulated_kernels_ros_gains_without_terrain_adaptation():
    worst, seen = run(64, 120, 32, KP_ROS, KD_ROS, 0)
    assert not seen["neg"] and not seen["pos"]


def test_fresh_state_is_the_reset_state_and_singular_plane_is_flat():
    B = 5
    state = E.swing_init(B)
    assert (state == 0.0).all()
    pos = np.zeros((3, B)); pos[2] = 0.3
    ref = np.full((9, B), 2.0)
    pitch = E.terrain_pitch(state, 1, pos, ref)
    assert (pitch == 0.0).all() and (ref[1] == 0.0).all()
    # first tick, all feet in stance: target = foot_pos_cur, and both velocities are the same difference against zero last positions
    sc = Scenario(B, 3)
    x = sc.tick()
    fk, con, cur, rc = E.swing_legs(state, CPS, DT, KP_RESET, KD_RESET, x["gait_counter"], x["plan_contacts"], x["rot_z"], x["foot_pos_abs"],
                                    x["foot_pos_target_rel"], x["foot_force"])
    assert con.tolist() == [15] * B and (fk == 0.0).all()
    assert np.array_equal(rc, x["foot_pos_abs"] / 60.0)        # one sample in a window of 60
    # a foot that starts in swing differentiates its Bezier target against zero: the reference's first-tick spike
    state = E.swing_init(B)
    gc = x["gait_counter"].copy(); gc[0] = 150.0
    fk, con, cur, rc = E.swing_legs(state, CPS, DT, KP_RESET, KD_RESET, gc, np.full(B, 14, dtype=np.uint32), x["rot_z"], x["foot_pos_abs"],
                                    x["foot_pos_target_rel"], x["foot_force"])
    assert con.tolist() == [14] * B and np.abs(fk[0:3]).max() > 1000.0 and (fk[3:] == 0.0).all()


def test_state_is_bound_to_its_batch_size():
    """robots do not share state: running robots 0..3 alone gives the same answer as inside a batch of 9"""
    sc = Scenario(9, 8)
    big, small = E.swing_init(9), E.swing_init(4)
    for t in range(40):
        x = sc.tick()
        keys = ("gait_counter", "plan_contacts", "rot_z", "foot_pos_abs", "foot_pos_target_rel", "foot_force")
        a = E.swing_legs(big, CPS, DT, KP_RESET, KD_RESET, *[x[k] for k in keys])
        b = E.swing_legs(small, CPS, DT, KP_RESET, KD_RESET, *[np.ascontiguousarray(x[k][..., :4]) for k in keys])
        assert np.array_equal(a[0][:, :4], b[0]) and np.array_equal(a[1][:4], b[1]) and np.array_equal(a[3][:, :4], b[3])
