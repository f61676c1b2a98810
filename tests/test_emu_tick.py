"""CPU: the two fused kernels of a control tick (tick_front_a, tick_front_b) on the block emulator against the staged kernels they fuse, on
the emulator too, with each side's own state: over 30 ticks of standstill -> walking -> toggled out and back, for the three adapter variants
and both stance modes (root_lin_vel_d from ref in MPC mode, from des in QP mode), every array the later stages read and every state buffer
bit-identical after every tick.  The estimator's rows of x0 and the terrain stage's row 1 of ref, which come from kernels outside the two, are
given the same values on both sides."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_command_py as EC  # noqa: E402
import emu_tick_py as E  # noqa: E402
from command_scenarios import DT  # noqa: E402
from tick_scenarios import tick_inputs  # noqa: E402


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


class Side:
    """the arrays and states of one side (dense [rows][B])"""

    def __init__(self, B, tp, imu_fields, cmd_fields):
        z = lambda r: np.zeros((r, B))
        self.rot, self.rz, self.x0, self.ia, self.ig = z(9), z(9), z(12), z(3), z(3)
        self.kpl, self.ref, self.des = z(3), z(9), z(12)
        self.fpr, self.jac, self.fvr, self.foot, self.fk, self.gc = z(12), z(36), z(12), z(12), z(12), z(4)
        self.mode, self.contacts = np.zeros(B, dtype=np.uint32), np.zeros(B, dtype=np.uint32)
        self.imu = z(imu_fields) if imu_fields else None
        self.cmd = z(cmd_fields)
        self.swing = z(E.swing_fields())

    def arrays(self):
        return {k: v for k, v in vars(self).items() if v is not None}


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("mode", ["mpc", "qp"])
def test_fused_kernels_bit_identical_to_staged_on_emulator(a1, variant, mode):
    B, T = 256, 30
    mpc = mode == "mpc"
    tp = a1.default_tick_params(variant, a1.TICK_MPC if mpc else a1.TICK_QP)
    seqs, speed = tick_inputs(B, T, 17 + variant)
    rng = np.random.default_rng(variant)
    cp = tp.command
    imu_fields = EC.imu_init(1).shape[0] if variant != a1.VARIANT_HARDWARE else 0
    sides = []
    for _ in range(2):
        s = Side(B, tp, imu_fields, EC.command_init(1, cp.variant, cp.body_height, cp.body_height_min, cp.body_height_max,
                                                    np.array(cp.kp_linear), np.array(cp.kp_linear_lock)).shape[0])
        if s.imu is not None:
            s.imu[:] = EC.imu_init(B)
        s.cmd[:] = EC.command_init(B, cp.variant, cp.body_height, cp.body_height_min, cp.body_height_max, np.array(cp.kp_linear),
                                   np.array(cp.kp_linear_lock), ref=s.ref if mpc else None)
        sides.append(s)
    plan, trel = np.zeros(B, dtype=np.uint32), np.zeros((12, B))
    walking = 0
    for t in range(T):
        est = np.concatenate([np.array([0.0, 0.0, 0.28])[:, None] + 0.02 * rng.standard_normal((3, B)), 0.3 * rng.standard_normal((3, B))])
        pitch = rng.uniform(-0.3, 0.3, B)
        for fused, s in zip((False, True), sides):
            s.x0[3:6], s.x0[9:12] = est[:3], est[3:]          # what the EKF leaves for this tick
            if mpc:
                s.ref[1] = pitch                                # what the terrain stage left in row 1
            E.front_a(fused, B, DT, seqs["quat"][t], seqs["gyro"][t], seqs["acc"][t], s.imu, s.rot, s.rz, s.x0, s.ia, s.ig, s.cmd, seqs["cmd"][t],
                      s.mode, s.kpl, s.ref if mpc else None, s.des)
            lvd = np.ascontiguousarray(s.ref[5:8] if mpc else s.des[6:9])
            E.front_b(fused, B, tp, DT, seqs["joint_pos"][t], seqs["joint_vel"][t], s.rot, s.rz, s.x0, lvd, s.mode, s.gc, speed, s.swing,
                      seqs["foot_force"][t], s.fpr, s.jac, s.fvr, s.foot, s.fk, s.contacts, plan=None if fused else plan, trel=None if fused else trel)
        a, b = sides[0].arrays(), sides[1].arrays()
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), (t, k)
        walking += int(sides[0].mode.sum())
    assert walking > 0 and (sides[0].mode == 0).any()
    assert (sides[0].contacts != 15).any() and np.abs(sides[0].fk).max() > 0
