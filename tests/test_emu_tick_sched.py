"""CPU: the front kernel of the scheduled tick (tick_front_sched) on the block emulator against the staged kernels it fuses, on the emulator
too: leg kinematics, update_plan with its schedule, swing legs, then schedule row 0 overwritten by the swing stage's contacts.  Over 30 ticks
of standstill -> walking -> toggled out and back (early contacts from foot forces of up to 80 N), for the three adapter variants in MPC mode,
at horizons 10 and 20, with the integer gait speeds of the other tick tests and with non-integer ones (the schedule's step st is the
threshold test fmod(c + st * speed, cpg) <= cps: with integer speeds every product is exact, so an FMA contracted differently in one kernel
would not show).  Every array the later stages read, every state buffer and the schedule are bit-identical after every tick.  The
estimator's rows of x0 and the terrain stage's row 1 of ref come from kernels outside the fused one and are given the same values on both
sides."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_command_py as EC  # noqa: E402
import emu_tick_py as E  # noqa: E402
import emu_tick_sched_py as ES  # noqa: E402
from command_scenarios import DT  # noqa: E402
from tick_scenarios import tick_inputs  # noqa: E402


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def gait_speeds(B, kind, seed):
    """[4][B] gait_counter_speed: tick_inputs' integer speeds, or one non-integer speed per robot in [1.5, 4.5]"""
    if kind == "integer":
        return None
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.repeat(rng.uniform(1.5, 4.5, B)[None, :], 4, axis=0))


def _popcount(m):
    return sum(((m >> i) & 1) for i in range(4))


@pytest.mark.parametrize("speeds", ["integer", "fractional"])
@pytest.mark.parametrize("N", [10, 20])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_sched_front_bit_identical_to_staged_on_emulator(a1, variant, N, speeds):
    B, T = 256, 30
    tp = a1.default_tick_params(variant, a1.TICK_MPC)
    tp.gait.horizon = N
    seqs, speed = tick_inputs(B, T, 23 + variant)
    sp = gait_speeds(B, speeds, 5 + variant)
    if sp is not None:
        speed = sp
    rng = np.random.default_rng(100 + variant)
    cp = tp.command
    imu_fields = EC.imu_init(1).shape[0] if variant != a1.VARIANT_HARDWARE else 0
    sides = []
    for _ in range(2):
        z = lambda r: np.zeros((r, B))
        s = dict(rot=z(9), rz=z(9), x0=z(12), ia=z(3), ig=z(3), kpl=z(3), ref=z(9), des=z(12), fpr=z(12), jac=z(36), fvr=z(12), foot=z(12),
                 fk=z(12), gc=z(4), mode=np.zeros(B, dtype=np.uint32), contacts=np.zeros(B, dtype=np.uint32),
                 sched=np.zeros((N, B), dtype=np.uint32), swing=z(ES.swing_fields()))
        s["imu"] = EC.imu_init(B) if imu_fields else None
        s["cmd"] = EC.command_init(B, cp.variant, cp.body_height, cp.body_height_min, cp.body_height_max, np.array(cp.kp_linear),
                                   np.array(cp.kp_linear_lock), ref=s["ref"])
        sides.append(s)
    plan, trel = np.zeros(B, dtype=np.uint32), np.zeros((12, B))
    census = dict(walking=0, early=0, four=0, three=0, standstill=0)
    for t in range(T):
        est = np.concatenate([np.array([0.0, 0.0, 0.28])[:, None] + 0.02 * rng.standard_normal((3, B)), 0.3 * rng.standard_normal((3, B))])
        pitch = rng.uniform(-0.3, 0.3, B)
        for fused, s in zip((False, True), sides):
            s["x0"][3:6], s["x0"][9:12] = est[:3], est[3:]      # what the EKF leaves for this tick
            s["ref"][1] = pitch                                 # what the terrain stage left in row 1
            E.front_a(fused, B, DT, seqs["quat"][t], seqs["gyro"][t], seqs["acc"][t], s["imu"], s["rot"], s["rz"], s["x0"], s["ia"], s["ig"],
                      s["cmd"], seqs["cmd"][t], s["mode"], s["kpl"], s["ref"], s["des"])
            lvd = np.ascontiguousarray(s["ref"][5:8])
            ES.front_sched(fused, B, tp, DT, N, seqs["joint_pos"][t], seqs["joint_vel"][t], s["rot"], s["rz"], s["x0"], lvd, s["mode"], s["gc"],
                           speed, s["swing"], seqs["foot_force"][t], s["fpr"], s["jac"], s["fvr"], s["foot"], s["fk"], s["contacts"], s["sched"],
                           plan=None if fused else plan, trel=None if fused else trel)
        a, b = sides
        for k in a:
            if a[k] is not None:
                assert a[k].tobytes() == b[k].tobytes(), (t, k)
        walk = a["mode"] != 0
        pc = _popcount(a["sched"])
        census["walking"] += int(walk.sum())
        census["early"] += int((a["contacts"] & ~plan != 0).sum())
        census["four"] += int(((pc[1:] == 4).any(axis=0) & walk).sum())
        census["three"] += int((pc == 3).any(axis=0).sum())
        census["standstill"] += int((a["sched"] == 15).all(axis=0).sum())
    print("variant %d N %d %s speeds: %s" % (variant, N, speeds, census))
    assert census["walking"] > 0 and (sides[0]["mode"] == 0).any()
    assert census["early"] > 0 and census["standstill"] > 0 and census["three"] > 0
    if N == 20 and speeds == "integer":
        assert census["four"] > 0     # a four-foot crossing step inside the window (an exact hit of the swing threshold)
