"""ekf_update_kernel on the CPU emulator (tests/emu) against the oracle, on the walking streams of ekf_scenarios.py: the NUMERICAL
contract for non-finite inputs with about two robots per warp, so that every warp's loop serves a poisoned robot next to another one,
and a short run past the first steady-state position-drift cut.  The emulator runs about 45 ms per robot-tick: the batches are
small.  test_gpu_ekf.py runs the same checks at full size on the GPU."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from ekf_scenarios import DT, RHO_FIX, RHO_OPT, numerical_contract, walk_against_oracle  # noqa: E402


@pytest.fixture(scope="module")
def E():
    import emu_py
    emu_py.lib()
    return emu_py


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


class EmuEkf:
    """the ekf_scenarios backend on the emulator: filter states are host arrays [B,342]; the lane order between collectives varies
    from tick to tick"""

    def __init__(self, E):
        self.E = E

    def kin(self, q, dq, rot):
        fpr, jac, fvr, fpa, fva = self.E.leg_kinematics(q, dq, rot, RHO_OPT.reshape(12), RHO_FIX.reshape(20))
        return fpr, fvr

    def init(self, fpr, rot):
        return self.E.ekf_init(fpr, rot)

    def update(self, h, flat, inp, fpr, fvr, tick):
        return self.E.ekf_update(h, DT, flat, inp["mode"], inp["acc"], inp["gyro"], inp["rot"], fpr, fvr, inp["force"], order=tick % 3)

    def state(self, h):
        return h.copy()

    def clone(self, h):
        return h.copy()


def test_non_finite_inputs_are_numerical_on_emulator(E, O):
    """24 robots (about two per warp): two of every poison kind of ekf_scenarios, among them a NaN foot force in walking mode, which
    must end NUMERICAL with the state untouched and contact bit 1 (fmax / fmin would turn it into a swing foot and update)"""
    plan, worst = numerical_contract(EmuEkf(E), O, 24, 1, seed=7, warm_ticks=3, per_kind=2, next_ticks=1)
    assert {k for k, b, row, v in plan} >= {"force_nan", "force_inf", "force_stand", "acc", "gyro", "rot", "fpr", "fvr"}
    print("\nemulated EKF NUMERICAL contract, 24 robots: worst |emu - oracle| %.3e" % worst)


def test_walk_past_the_first_steady_state_cut_on_emulator(E, O):
    """two robots, 335 ticks: the cut of ticks 0-2, then the first one of the steady state (P[0,0] grown back) agrees with the oracle"""
    worst, cuts = walk_against_oracle(EmuEkf(E), O, 2, 335, 0, seed=5)
    assert cuts[:3].all() and cuts[300:].any(axis=0).all(), [np.nonzero(cuts[:, b])[0].tolist() for b in range(2)]
    assert worst <= 1e-10, worst
    print("\nemulated EKF 2 robots x 335 ticks: worst |emu - oracle| %.3e, cut ticks %s" % (worst, [np.nonzero(cuts[:, b])[0].tolist() for b in range(2)]))
