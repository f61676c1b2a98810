"""GPU tests of the scheduled tick (a1mpc_tick_* in MPC mode with gait.horizon = the handle's horizon): the solve poses update_plan's
contact schedule, step 0 replaced by the swing stage's contacts, instead of the current contacts held over the horizon.
  * Every output of every tick bit-identical to the hand-built chain of staged entry points with the schedule (staged_chain_sched below:
    tests/tick_scenarios.py's chain with update_plan writing the schedule, the swing stage's contacts copied into its row 0, then
    a1mpc_solve_batch_ext_warm with shift 1 at horizon 10 or a1mpc_solve_batch_ext at horizon 20): the three adapter variants at B = 1024
    over 30 ticks, non-integer gait speeds, B = 65 536, host = device arrays, reset, horizon 20; on the default handle (two-feet schedules
    go to the compacted kernel) and on an A1MPC_EXT_COMPACT=0 handle (every robot on the general kernel).
  * Against the oracle: the tick on the raw inputs of tests/sched_tick_scenarios.py's closed loop (B = 512 x 64 ticks at horizon 10, and
    a smaller run at horizon 20), every QP OPTIMAL and within 1e-4 N of the oracle's exact solve of that run's `early` variant, contacts
    and modes exact, x0 within 1e-8, torques as in test_gpu_sched_tick.py's device loop.
  * Argument errors: gait.horizon other than 0 or the handle's horizon is rejected in MPC mode and ignored in QP mode."""
import ctypes as C
import os

import numpy as np
import pytest

from command_scenarios import DT
from common import obatch
from sched_tick_scenarios import describe, stacked, tick_solve_inputs
from swing_scenarios import KD_ROS, KP_ROS
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, off, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)
TOL_LOOP = 1e-4     # N: the device chain's x0 matches the oracle chain's to 1e-8 only (test_gpu_sched_tick.py)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def _engine(a1, horizon=10, compact=True):
    if compact:
        return a1.Engine(a1.default_config(horizon=horizon))
    os.environ["A1MPC_EXT_COMPACT"] = "0"
    try:
        return a1.Engine(a1.default_config(horizon=horizon))
    finally:
        del os.environ["A1MPC_EXT_COMPACT"]


@pytest.fixture(scope="module", params=[True, False], ids=["routed", "general_only"])
def eng(a1, request):
    e = _engine(a1, 10, request.param)
    yield e
    e.close()


def sched_params(a1, variant, N):
    tp = a1.default_tick_params(variant, a1.TICK_MPC)
    tp.gait.horizon = N
    return tp


def staged_chain_sched(a1, eng, tp, ds, B, T, dt):
    """the scheduled tick's stages as separate entry points on device pointers (MPC mode), from the same start state as a1mpc_tick_create:
    tick_scenarios.staged_chain with update_plan's schedule d_sched, the swing stage's contacts copied into row 0 (through the host: the
    C ABI has no device-to-device copy), then a1mpc_solve_batch_ext_warm (shift 1) at horizon 10 or a1mpc_solve_batch_ext at horizon 20,
    world-z pyramids; one dict of host outputs per tick"""
    L = a1.lib()
    N = eng.cfg.horizon
    assert tp.mode == a1.TICK_MPC and tp.gait.horizon == N
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status")}
    d_sched = eng.dalloc(N * B * 4)
    imu = eng.imu_alloc(B) if tp.command.variant != a1.VARIANT_HARDWARE else None
    sw, ekf = eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B))
    warm = eng.warm_alloc(B) if N == 10 else None
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), dv["ref"], B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    inp = a1.Inputs(dv["x0"], dv["rot"], dv["foot"], dv["ref"], u["contact"], B)
    out = a1.Outputs(dv["f_body"], u["status"], None, None, B)
    ext = a1.InputsExt(d_sched.value, None)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    res = []
    for t in range(T):
        a1._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                            dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                               rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, dt, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], dv["ref"], B, dv["des"], B))
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(tp.gait), dv["gc"], ds.speed, u["mode"], x0p(9), off(dv["ref"], 5 * B * 8), dv["rz"],
                                            dv["rot"], x0p(3), u["plan"], d_sched, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"], dv["rz"],
                                           dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        h2d(a1, eng, d_sched, d2h(a1, eng, u["contact"], B, np.uint32))      # row 0 of the schedule
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                               ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
        if warm is not None:
            a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out), warm, 1))
        else:
            a1._check(L.a1mpc_solve_batch_ext(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out)))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        src = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"], ref=dv["ref"])
        res.append({k: d2h(a1, eng, src[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS})
    for p in list(dv.values()) + list(u.values()) + [d_sched, imu, sw, ekf, warm, cs]:
        if p is not None:
            L.a1mpc_device_free(eng.h, p)
    return res


def fractional_speeds(B, seed):
    """[4][B] gait_counter_speed, one non-integer speed per robot: the schedule's threshold products are then not exact"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.repeat(rng.uniform(1.5, 4.5, B)[None, :], 4, axis=0))


def _compare(a1, eng, tp, B, T, seed, speed=None):
    seqs, sp = tick_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, sp if speed is None else speed)
    try:
        want = staged_chain_sched(a1, eng, tp, ds, B, T, DT)
        tick = a1.Tick(eng, B, tp)
        try:
            got = tick_run_device(a1, eng, tick, ds, B, T, DT)
        finally:
            tick.close()
    finally:
        ds.free()
    return got, want


def _status_counts(got):
    return [np.bincount(g["status"], minlength=5).tolist() for g in got]


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_sched_tick_bit_identical_to_staged_chain(a1, eng, variant):
    B, T = 1024, 30
    got, want = _compare(a1, eng, sched_params(a1, VARIANTS[variant], 10), B, T, seed=61 + VARIANTS[variant])
    assert first_difference(got, want) is None, first_difference(got, want)
    modes = np.array([g["movement_mode"] for g in got])
    assert modes[:5].sum() == 0 and modes[5:].sum() > 0 and (modes[-1] == 0).any()     # standstill, walking, toggled out
    print("%s: %d ticks bit-identical, status per tick %s" % (variant, T, _status_counts(got)))


def test_fractional_gait_speeds_bit_identical(a1, eng):
    B, T = 1024, 30
    got, want = _compare(a1, eng, sched_params(a1, a1.VARIANT_GAZEBO, 10), B, T, seed=71, speed=fractional_speeds(B, 72))
    assert first_difference(got, want) is None, first_difference(got, want)


def test_large_batch_bit_identical(a1, eng):
    B, T = 65536, 3
    got, want = _compare(a1, eng, sched_params(a1, a1.VARIANT_GAZEBO, 10), B, T, seed=11)
    assert first_difference(got, want) is None, first_difference(got, want)
    print("B=%d scheduled: status counts per tick %s" % (B, _status_counts(got)))


def test_host_and_device_arrays_agree(a1, eng):
    B, T = 256, 8
    tp = sched_params(a1, a1.VARIANT_GAZEBO, 10)
    seqs, speed = tick_inputs(B, T, 7)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    tick = a1.Tick(eng, B, tp)
    try:
        dev = tick_run_device(a1, eng, tick, ds, B, T, DT)
        tick.reset()
        host = []
        for t in range(T):
            tau, o = tick.run(DT, *(seqs[k][t] for k in a1.TICK_INPUTS[:-1]), speed)
            o["tau"] = tau
            host.append(o)
    finally:
        tick.close()
        ds.free()
    assert first_difference(host, dev) is None, first_difference(host, dev)


def test_reset_reproduces_the_first_ticks(a1, eng):
    B, T = 512, 12
    tp = sched_params(a1, a1.VARIANT_ISAAC, 10)
    seqs, speed = tick_inputs(B, T, 3)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    tick = a1.Tick(eng, B, tp)
    try:
        first = tick_run_device(a1, eng, tick, ds, B, T, DT)
        tick.reset()
        again = tick_run_device(a1, eng, tick, ds, B, T, DT)
    finally:
        tick.close()
        ds.free()
    assert first_difference(again, first) is None, first_difference(again, first)


def test_horizon_20_cold_solve(a1):
    e = _engine(a1, 20)
    try:
        got, want = _compare(a1, e, sched_params(a1, a1.VARIANT_GAZEBO, 20), 256, 30, seed=5)
    finally:
        e.close()
    assert first_difference(got, want) is None, first_difference(got, want)
    print("horizon 20 scheduled: status per tick %s" % _status_counts(got))


def test_argument_errors(a1):
    L = a1.lib()
    B = 64
    e = _engine(a1, 10)
    t = C.c_void_p()
    try:
        for horizon in (5, 20, -1):
            tp = sched_params(a1, a1.VARIANT_GAZEBO, horizon)
            assert L.a1mpc_tick_create(e.h, B, C.byref(tp), C.byref(t)) == -1 and b"gait.horizon" in L.a1mpc_last_error(), horizon
        # QP mode ignores gait.horizon: the same outputs as with 0
        seqs, speed = tick_inputs(B, 4, 9)
        outs = []
        for horizon in (0, 5):
            tp = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP)
            tp.gait.horizon = horizon
            tick = a1.Tick(e, B, tp)
            try:
                res = []
                for k in range(4):
                    tau, o = tick.run(DT, *(seqs[n][k] for n in a1.TICK_INPUTS[:-1]), speed)
                    o["tau"] = tau
                    res.append(o)
                outs.append(res)
            finally:
                tick.close()
        assert first_difference(outs[1], outs[0]) is None
        # after the rejected creates the handle still serves a scheduled tick
        tick = a1.Tick(e, B, sched_params(a1, a1.VARIANT_GAZEBO, 10))
        try:
            tau, o = tick.run(DT, *(seqs[n][0] for n in a1.TICK_INPUTS[:-1]), speed)
        finally:
            tick.close()
        assert np.isfinite(tau).all() and (o["status"] == a1.STATUS_OPTIMAL).all()
    finally:
        e.close()


# ---- against the oracle: the closed loop of tests/sched_tick_scenarios.py -------------------------------------------------------------

def _oracle_loop(a1, O, B, T, seed, N):
    """the scheduled tick on the raw inputs of sched_tick_scenarios.tick_solve_inputs, with that chain's gains and leg geometry, against the
    oracle chain and the oracle's exact solve of its `early` variant (schedule step 0 = the swing stage's contacts)"""
    D = tick_solve_inputs(B, T, seed, N)
    st, sched, _ = stacked(D, "early")
    fo_all, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, st), sched, None, O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (info[:, 1] == 1).all()
    tp = sched_params(a1, a1.VARIANT_GAZEBO, N)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    tp.rho_opt[:], tp.rho_fix[:] = D["rho_opt"].tolist(), D["rho_fix"].tolist()
    tp.kp_foot[:], tp.kd_foot[:], tp.km_foot[:], tp.torques_gravity[:] = KP_ROS.tolist(), KD_ROS.tolist(), km.tolist(), tg.tolist()
    tp.use_terrain_adapt, tp.assume_flat_ground = 1, 1
    eng = _engine(a1, N)
    ds = DeviceSeqs(a1, eng, D["seqs"], D["speed"])
    tick = a1.Tick(eng, B, tp)
    try:
        got = tick_run_device(a1, eng, tick, ds, B, T, DT)
    finally:
        tick.close()
        ds.free()
        eng.close()
    tau0 = np.zeros((12, B))
    worst = dict(f=0.0, tau=0.0, x0=0.0)
    for t, g in enumerate(got):
        fo = fo_all[:, t * B:(t + 1) * B]
        for b in range(B):
            tau0[:, b] = O.joint_torques(fo[:, b], D["fk"][t][:, b], D["jac"][t][:, b], int(D["contact"][t][b]), km, tg, tau0[:, b])
        assert np.array_equal(g["movement_mode"], D["mode"][t]) and np.array_equal(g["contacts"], D["contact"][t]), t
        ex = float(np.abs(g["x0"] - D["x0"][t]).max())
        assert ex <= 1e-8, (t, ex)
        ef = np.abs(g["f_body"] - fo).max(axis=0)
        bad = np.nonzero((g["status"] != a1.STATUS_OPTIMAL) | ~(ef <= TOL_LOOP))[0]
        assert bad.size == 0, "scheduled tick N=%d, tick %d: %d QPs fail (status %s, |f - f*| %s)\n%s" % (
            N, t, bad.size, g["status"][bad][:8].tolist(), ef[bad][:8].tolist(), describe(D, "early", t * B + bad))
        jn = np.abs(D["jac"][t].T.reshape(B, 4, 3, 3)).sum(axis=2).reshape(B, 12).T
        et = float((np.abs(g["tau"] - tau0) - (1e-4 * jn + 1e-8 * np.maximum(1.0, np.abs(tau0)))).max())
        assert et <= 0.0, (t, et)
        worst = dict(f=max(worst["f"], float(ef.max())), tau=max(worst["tau"], float(np.abs(g["tau"] - tau0).max())), x0=max(worst["x0"], ex))
    print("scheduled tick vs oracle, N=%d, B=%d x %d ticks: |x0 - x0_oracle| %.2e, |f - f_oracle| %.2e N, |tau - tau_oracle| %.2e Nm" % (
        N, B, T, worst["x0"], worst["f"], worst["tau"]))


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def test_against_oracle_horizon_10(a1, O):
    _oracle_loop(a1, O, 512, 64, 43, 10)


def test_against_oracle_horizon_20(a1, O):
    _oracle_loop(a1, O, 128, 64, 43, 20)
