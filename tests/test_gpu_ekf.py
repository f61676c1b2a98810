"""GPU: the batched Kalman filter (a1mpc_ekf_update_batch, ekf_update_kernel) against the oracle's restatement of A1BasicEKF on the
walking streams of ekf_scenarios.py, each side carrying its own filter state from tick to tick.

* Long runs: 2000 ticks, with and without assume_flat_ground.  The position-drift cut (A1BasicEKF.cpp:144-148) fires on the first
  ticks from P = 3 I and again only once P[0,0] has grown back, about 300 ticks later: only a run that long reaches the filter's
  steady state.  Every tick compares x, P, the outputs and the cut decision of every robot.
* Multi-robot warps: the kernel's grid stops at 2 x SMs blocks of 4 warps (1056 robots on 132 SMs), and each warp then loops over
  several robots through the same shared memory.  B = 4099 gives every warp 3 or 4 robots and leaves the last pass partial.
* The NUMERICAL contract for non-finite inputs (ekf_scenarios.numerical_contract), at B = 4099 so that poisoned robots share their
  warps with healthy ones, and through a whole control tick."""
import numpy as np
import pytest

from ekf_scenarios import DT, RHO_FIX, RHO_OPT, numerical_contract, walk_against_oracle
from tick_scenarios import tick_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def eng(a1):
    e = a1.Engine(a1.default_config(horizon=10))
    yield e
    e.close()


class GpuEkf:
    """the ekf_scenarios backend on the C ABI: leg kinematics, filter states in device memory"""

    def __init__(self, a1, eng):
        self.a1, self.eng, self.bufs = a1, eng, []

    def kin(self, q, dq, rot):
        fpr, jac, fvr, fpa, fva = self.eng.leg_kinematics(q, dq, rot, RHO_OPT.reshape(12), RHO_FIX.reshape(20))
        return fpr, fvr

    def _alloc(self, B):
        p = self.eng.ekf_alloc(B)
        self.bufs.append(p)
        return p, B

    def init(self, fpr, rot):
        h = self._alloc(fpr.shape[1])
        self.eng.ekf_init(h[0], fpr, rot)
        return h

    def update(self, h, flat, inp, fpr, fvr, tick):
        return self.eng.ekf_update(h[0], DT, flat, inp["mode"], inp["acc"], inp["gyro"], inp["rot"], fpr, fvr, inp["force"])

    def state(self, h):
        x, P = self.eng.ekf_state(*h)
        return np.ascontiguousarray(np.concatenate([x, P.reshape(h[1], 324)], axis=1))

    def clone(self, h):
        s = self.state(h)
        c = self._alloc(h[1])
        self.a1._check(self.a1.lib().a1mpc_memcpy_h2d(self.eng.h, c[0], s.ctypes.data, s.nbytes))
        self.eng.sync()
        return c

    def free(self):
        for p in self.bufs:
            self.a1.lib().a1mpc_device_free(self.eng.h, p)
        self.bufs = []


@pytest.fixture
def dev(a1, eng):
    d = GpuEkf(a1, eng)
    yield d
    d.free()


@pytest.mark.parametrize("flat", [0, 1])
def test_long_walk_against_oracle(dev, O, flat):
    B, T = 256, 2000
    worst, cuts = walk_against_oracle(dev, O, B, T, flat, seed=5 + flat)
    late = cuts[300:].any(axis=0)
    first = 300 + cuts[300:].argmax(axis=0)[late]
    print("\nEKF %d robots x %d ticks, assume_flat_ground %d: worst |gpu - oracle| %.3e; cut on ticks 0-2 on %d robots, again after tick 300 "
          "on %d robots (%d robot-ticks), first such tick %s" % (B, T, flat, worst, cuts[:3].all(axis=0).sum(), late.sum(), cuts[300:].sum(),
                                                                "%d-%d" % (first.min(), first.max()) if late.any() else "-"))
    assert worst <= 1e-10, worst
    assert cuts[:3].all()
    # steady state: P[0,0] grows back to the cut's threshold and the cut fires again on almost every robot
    assert late.sum() >= 0.9 * B, late.sum()


def test_multi_robot_warps_against_oracle(dev, O):
    import torch
    B, T = 4099, 60
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert B > 3 * (2 * sms) * 4, "fewer than three robots per warp on %d SMs" % sms
    worst, cuts = walk_against_oracle(dev, O, B, T, 1, seed=21)
    print("\nEKF B = %d (%.2f robots per warp on %d SMs), %d ticks: worst |gpu - oracle| %.3e" % (B, B / (8.0 * sms), sms, T, worst))
    assert worst <= 1e-10, worst


@pytest.mark.parametrize("flat", [0, 1])
def test_non_finite_inputs_are_numerical_and_leave_the_state(dev, O, flat):
    plan, worst = numerical_contract(dev, O, 4099, flat, seed=31 + flat, warm_ticks=6, per_kind=12)
    print("\nEKF NUMERICAL contract, B = 4099, %d poisoned robots, assume_flat_ground %d: worst |gpu - oracle| %.3e" % (len(plan), flat, worst))


@pytest.mark.parametrize("mode", ["mpc", "qp"])
def test_tick_keeps_the_estimate_of_a_robot_with_a_nan_foot_force(a1, eng, mode):
    """a NaN foot force in walking mode makes that robot's EKF update NUMERICAL inside a1mpc_tick_run: its x0 rows 3-5 (root
    position) and 9-11 (root velocity) keep the previous tick's estimate, and every output of every other robot is bit-identical to
    the run without the NaN"""
    B, T, tp, r, leg = 64, 14, 11, 37, 2
    seqs, speed = tick_inputs(B, T, seed=3)
    params = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC if mode == "mpc" else a1.TICK_QP)

    def run(force):
        tick = a1.Tick(eng, B, params)
        try:
            outs = []
            for t in range(T):
                args = {k: seqs[k][t] for k in ("quat", "gyro", "acc", "joint_pos", "joint_vel", "cmd")}
                outs.append(tick.run(DT, foot_force=force[t], gait_counter_speed=speed, **args)[1])
            return outs
        finally:
            tick.close()

    clean = run(seqs["foot_force"])
    poisoned_force = seqs["foot_force"].copy()
    poisoned_force[tp, leg, r] = np.nan
    got = run(poisoned_force)
    assert clean[tp]["movement_mode"][r] == 1
    for t in range(tp):
        for k in clean[t]:
            assert got[t][k].tobytes() == clean[t][k].tobytes(), (t, k)
    rows = [3, 4, 5, 9, 10, 11]
    assert got[tp]["x0"][rows, r].tobytes() == got[tp - 1]["x0"][rows, r].tobytes()
    assert np.isfinite(got[tp]["x0"][:, r]).all()
    assert clean[tp]["x0"][rows, r].tobytes() != clean[tp - 1]["x0"][rows, r].tobytes()
    others = np.arange(B) != r
    for k in clean[tp]:
        assert got[tp][k][..., others].tobytes() == clean[tp][k][..., others].tobytes(), k
