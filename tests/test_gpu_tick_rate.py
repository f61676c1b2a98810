"""GPU tests of a tick whose MPC solve runs at a lower rate than the tick (a1mpc_tick_set_mpc_period) and of its staged entry point
a1mpc_plan_forces_batch.
  1. Every output of every run is bit-identical to a staged chain (staged_chain_rate below): the chain of tests/tick_scenarios.py, or of the
     scheduled or terrain ticks, whose solve gathers the robots that are due by the rule (n == 0 or n % period == b % period) and their warm
     slots into a dense sub-batch, solves it with a1mpc_solve_batch_warm / _ext_warm / _ext / a1mpc_solve_batch asking for u_full, scatters
     the results back, and then calls a1mpc_plan_forces_batch (PLAN) and the torques.  Three variants x {held, scheduled} x {HOLD, PLAN} x
     periods {2, 4, N} at B = 1024 over 40 runs; horizon 20 held and scheduled at period 4; ESTIMATED terrain on both ticks; B = 65 536.
  2. Period 1, never set or set back, is the plain tick bit for bit; switching the period mid-run (1 -> 4 -> 2 -> 1) makes every robot
     solve on the next run (the chain switching alike); reset_robots of 25 % mid-walk makes the masked robots solve on their next run as a
     period-1 tick with the same reset does, and leaves every other robot's outputs as without the reset; a1mpc_tick_reset repeats the
     first runs; host arrays give the device arrays' results; argument errors.
  3. Against the oracle: the due robots' QPs of the chain's closed loop of tests/sched_tick_scenarios.tick_solve_inputs (seed 43,
     B = 512 x 64 runs, N = 10, period 4) are every one OPTIMAL and within 1e-4 N of compute_grf_batch / compute_grf_batch_ext."""
import ctypes as C

import numpy as np
import pytest

from command_scenarios import DT
from common import obatch
from sched_tick_scenarios import tick_solve_inputs
from swing_scenarios import KD_ROS, KP_ROS
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, off, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)
FLAT, ESTIMATED = 0, 1
HOLD, PLAN = 0, 1
TOL_ORACLE = 1e-4   # N: the tolerance of the scheduled tick against the oracle (test_gpu_tick_sched.py)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def engines(a1):
    es = {10: a1.Engine(a1.default_config(horizon=10)), 20: a1.Engine(a1.default_config(horizon=20))}
    yield es
    for e in es.values():
        e.close()


def _params(a1, variant, kind, N):
    tp = a1.default_tick_params(variant, a1.TICK_MPC)
    if kind == "sched":
        tp.gait.horizon = N
    return tp


def due_rule(n, period):
    return (n == 0) | (n % period == np.arange(n.shape[0]) % period)


def staged_chain_rate(a1, eng, tp, ds, B, T, dt, periods, playback, source=FLAT, record=False):
    """the multi-rate tick as separate entry points on device pointers (MPC mode), from the same start state as a1mpc_tick_create.
    periods[t]: the period of run t (a change makes every robot solve on that run); the robots due at run t are solved as one dense
    sub-batch through host arrays: warm with shift 0 on the held pattern, shift = period on the schedule, cold at horizon 20; source
    ESTIMATED poses the pyramids on a1mpc_terrain_normals_batch's normals (the held pattern as the swing stage's contacts in all N rows).
    One dict of host outputs per run; with record also the due mask, the sub-batch's iterations and the solve's inputs of every robot."""
    L = a1.lib()
    N = eng.cfg.horizon
    sched_tick = tp.gait.horizon == N
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12, nrm=12,
              plan=12 * N)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status", "step")}
    d_sched = eng.dalloc(N * B * 4)
    imu = eng.imu_alloc(B) if tp.command.variant != a1.VARIANT_HARDWARE else None
    sw, ekf = eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B))
    warm = eng.warm_alloc(B) if N == 10 else None
    W = (L.a1mpc_warm_bytes(eng.h, B) // 4) // B if warm is not None else 0
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), dv["ref"], B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    f_body, status, plan = np.zeros((12, B)), np.zeros(B, np.int32), np.zeros((12 * N, B))
    n, j = np.zeros(B, np.int64), np.zeros(B, np.int64)
    res = []
    for t in range(T):
        p = periods[t]
        if t > 0 and p != periods[t - 1]:
            n[:], j[:] = 0, 0
        a1._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                            dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                               rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, dt, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], dv["ref"], B, dv["des"], B))
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(tp.gait), dv["gc"], ds.speed, u["mode"], x0p(9), off(dv["ref"], 5 * B * 8), dv["rz"],
                                            dv["rot"], x0p(3), u["plan"], d_sched if sched_tick else None, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"], dv["rz"],
                                           dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        con = d2h(a1, eng, u["contact"], B, np.uint32)
        if sched_tick:
            h2d(a1, eng, d_sched, con)                                           # row 0 of the schedule
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                               ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        if source == FLAT:
            a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
        else:
            a1._check(L.a1mpc_terrain_normals_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None, dv["nrm"]))
        # the solve of the due robots, as one dense sub-batch
        due = due_rule(n, p)
        idx = np.nonzero(due)[0]
        st = {k: d2h(a1, eng, dv[k], (r, B)) for k, r in (("x0", 12), ("rot", 9), ("foot", 12), ("ref", 9))}
        st["contact"] = con
        sc = d2h(a1, eng, d_sched, (N, B), np.uint32) if sched_tick else np.tile(con, (N, 1))
        nm = d2h(a1, eng, dv["nrm"], (12, B)) if source != FLAT else None
        sub = {k: np.ascontiguousarray(v[..., idx]) for k, v in st.items()}
        iters = None
        if idx.size:
            wsub = None
            if warm is not None:
                wall = d2h(a1, eng, warm, (B, W), np.uint32)
                wsub = eng.dalloc(idx.size * W * 4)
                h2d(a1, eng, wsub, wall[idx])
            ext = None
            if sched_tick or source != FLAT:
                ext = (np.ascontiguousarray(sc[:, idx]), np.ascontiguousarray(nm[:, idx]) if nm is not None else None)
            shift = p if sched_tick else 0
            if warm is not None and ext is not None:
                fs, ss, iters, us = eng._solve(L.a1mpc_solve_batch_ext_warm, sub, True, ext=ext, warm_args=(wsub, shift))
            elif warm is not None:
                fs, ss, iters, us = eng._solve(L.a1mpc_solve_batch_warm, sub, True, warm_args=(wsub, 0))
            elif ext is not None:
                fs, ss, iters, us = eng._solve(L.a1mpc_solve_batch_ext, sub, True, ext=ext)
            else:
                fs, ss, iters, us = eng._solve(L.a1mpc_solve_batch, sub, True)
            if wsub is not None:
                wall[idx] = d2h(a1, eng, wsub, (idx.size, W), np.uint32)
                h2d(a1, eng, warm, wall)
                L.a1mpc_device_free(eng.h, wsub)
            f_body[:, idx], status[idx], plan[:, idx] = fs, ss, us
        j = np.where(due, 0, j + 1)
        n += 1
        h2d(a1, eng, dv["f_body"], f_body)
        h2d(a1, eng, u["status"], status)
        if playback == PLAN and p > 1:
            h2d(a1, eng, dv["plan"], plan)
            h2d(a1, eng, u["step"], j.astype(np.uint32))
            a1._check(L.a1mpc_plan_forces_batch(eng.h, B, dv["rot"], dv["plan"], u["step"], dv["f_body"]))
            f_body = d2h(a1, eng, dv["f_body"], (12, B))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        srcs = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"], ref=dv["ref"])
        r = {k: d2h(a1, eng, srcs[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS}
        if record:
            r.update(due=due, iters=iters, sched=sc, normals=nm, **{k: st[k] for k in ("rot", "foot")})
        res.append(r)
    for q in list(dv.values()) + list(u.values()) + [d_sched, imu, sw, ekf, warm, cs]:
        if q is not None:
            L.a1mpc_device_free(eng.h, q)
    return res


def tick_run_rate(a1, eng, tp, ds, B, T, dt, periods, playback, source=FLAT, resets=None, full_reset_at=None, setup=None):
    """runs 0 .. T-1 of a fresh tick on device pointers; set_mpc_period(periods[t], playback) before run t whenever the period changes (and
    before run 0 unless it is None: never set); resets {t: mask}: reset_robots_ptr before run t; full_reset_at: a1mpc_tick_reset before that
    run; setup(tick) after create.  One dict per run."""
    L = a1.lib()
    d = {k: eng.dalloc(int(np.prod(OUT_SPECS[k][0] + (B,))) * np.dtype(OUT_SPECS[k][1]).itemsize) for k in OUT_SPECS}
    outs = a1.TickOutputs(*[d.get(k) for k in a1.TICK_OUTPUTS])
    d_mask = eng.dalloc(B)
    tick = a1.Tick(eng, B, tp)
    if source != FLAT:
        tick.set_terrain(source)
    if setup:
        setup(tick)
    res, cur = [], None
    try:
        for t in range(T):
            if periods[t] is not None and periods[t] != cur:
                tick.set_mpc_period(periods[t], playback)
                cur = periods[t]
            if resets and t in resets:
                h2d(a1, eng, d_mask, np.ascontiguousarray(resets[t], dtype=np.uint8))
                tick.reset_robots_ptr(d_mask.value)
            if full_reset_at == t:
                tick.reset()
            ins = a1.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1.TICK_INPUTS])
            tick.run_ptrs(dt, ins, outs)
            res.append({k: d2h(a1, eng, d[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS})
    finally:
        tick.close()
        for q in list(d.values()) + [d_mask]:
            L.a1mpc_device_free(eng.h, q)
    return res


def _compare(a1, eng, tp, B, T, seed, periods, playback, source=FLAT):
    seqs, speed = tick_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        want = staged_chain_rate(a1, eng, tp, ds, B, T, DT, periods, playback, source)
        got = tick_run_rate(a1, eng, tp, ds, B, T, DT, periods, playback, source)
    finally:
        ds.free()
    return got, want


# ---- 1. the tick against the staged chain ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("period", [2, 4, 10])
@pytest.mark.parametrize("playback", [HOLD, PLAN], ids=["hold", "plan"])
@pytest.mark.parametrize("kind", ["held", "sched"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_tick_bit_identical_to_staged_chain(a1, engines, variant, kind, playback, period):
    eng = engines[10]
    B, T = 1024, 40
    got, want = _compare(a1, eng, _params(a1, VARIANTS[variant], kind, 10), B, T, 71 + VARIANTS[variant], [period] * T, playback)
    assert first_difference(got, want) is None, first_difference(got, want)
    moved = sum(int((g["f_body"] != got[t - 1]["f_body"]).any(axis=0).sum()) for t, g in enumerate(got) if t > 0)
    print("%s %s period %d %s: %d runs bit-identical, robots whose forces changed per run %.0f" % (
        variant, kind, period, "plan" if playback else "hold", T, moved / (T - 1)))


@pytest.mark.parametrize("source", [FLAT, ESTIMATED], ids=["flat", "estimated"])
@pytest.mark.parametrize("kind", ["held", "sched"])
@pytest.mark.parametrize("N", [10, 20])
def test_horizon_and_terrain_bit_identical(a1, engines, N, kind, source):
    if N == 10 and source == FLAT:
        pytest.skip("covered by test_tick_bit_identical_to_staged_chain")
    eng = engines[N]
    B, T = 1024, 24
    got, want = _compare(a1, eng, _params(a1, a1.VARIANT_GAZEBO, kind, N), B, T, 81, [4] * T, PLAN, source)
    assert first_difference(got, want) is None, first_difference(got, want)


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_large_batch_bit_identical(a1, engines, kind):
    B, period = 65536, 4
    T = 2 * period
    got, want = _compare(a1, engines[10], _params(a1, a1.VARIANT_GAZEBO, kind, 10), B, T, 11, [period] * T, PLAN)
    assert first_difference(got, want) is None, first_difference(got, want)


def test_plan_forces_batch_host_and_device(a1, engines):
    eng = engines[10]
    L = a1.lib()
    B, N = 1000, 10
    rng = np.random.default_rng(3)
    rot, u, f0 = rng.standard_normal((9, B)), rng.standard_normal((12 * N, B)), rng.standard_normal((12, B))
    step = rng.integers(0, N + 2, B).astype(np.uint32)
    fh = eng.plan_forces(rot, u, step, f0)
    d = {k: eng.dalloc(a.nbytes) for k, a in dict(rot=rot, u=u, step=step, f=f0).items()}
    try:
        for k, a in dict(rot=rot, u=u, step=step, f=f0).items():
            h2d(a1, eng, d[k], a)
        a1._check(L.a1mpc_plan_forces_batch(eng.h, B, d["rot"], d["u"], d["step"], d["f"]))
        fd = d2h(a1, eng, d["f"], (12, B))
    finally:
        for q in d.values():
            L.a1mpc_device_free(eng.h, q)
    assert fh.tobytes() == fd.tobytes()
    R = rot.reshape(3, 3, B)
    us = u.reshape(N, 4, 3, B)[np.minimum(step, N - 1), :, :, np.arange(B)]
    want = np.where(step >= N, 0.0, np.einsum("kab,blk->lab", R, us).reshape(12, B))
    want = np.where(step == 0, f0, want)
    assert np.abs(fh - want).max() <= 1e-13


# ---- 2. compatibility and state --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["held", "sched"])
def test_period_one_is_the_plain_tick(a1, engines, kind):
    eng = engines[10]
    B, T = 1024, 20
    tp = _params(a1, a1.VARIANT_GAZEBO, kind, 10)
    seqs, speed = tick_inputs(B, T, 21)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        plain = tick_run_device(a1, eng, a1.Tick(eng, B, tp), ds, B, T, DT)
        one = tick_run_rate(a1, eng, tp, ds, B, T, DT, [1] * T, PLAN)
        back = tick_run_rate(a1, eng, tp, ds, B, T, DT, [None] * T, PLAN,
                             setup=lambda tick: (tick.set_mpc_period(4, a1.PLAYBACK_PLAN), tick.set_mpc_period(1, a1.PLAYBACK_HOLD)))
    finally:
        ds.free()
    assert first_difference(one, plain) is None
    assert first_difference(back, plain) is None


def test_switching_the_period_mid_run(a1, engines):
    eng = engines[10]
    B, T = 1024, 32
    periods = [1] * 6 + [4] * 10 + [2] * 8 + [1] * 8
    for kind in ("held", "sched"):
        got, want = _compare(a1, eng, _params(a1, a1.VARIANT_GAZEBO, kind, 10), B, T, 31, periods, PLAN)
        assert first_difference(got, want) is None, (kind, first_difference(got, want))


def test_reset_robots_mid_walk(a1, engines):
    eng = engines[10]
    B, T, t_r, period = 1024, 30, 13, 4
    tp = _params(a1, a1.VARIANT_GAZEBO, "held", 10)
    seqs, speed = tick_inputs(B, T, 41)
    mask = np.random.default_rng(4).random(B) < 0.25
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        walk = tick_run_rate(a1, eng, tp, ds, B, T, DT, [period] * T, PLAN)
        reset = tick_run_rate(a1, eng, tp, ds, B, T, DT, [period] * T, PLAN, resets={t_r: mask})
        plain = tick_run_rate(a1, eng, tp, ds, B, T, DT, [1] * T, PLAN, resets={t_r: mask})
    finally:
        ds.free()
    for t in range(T):
        for k in OUT_SPECS:
            g, w = reset[t][k], walk[t][k]
            assert g[..., ~mask].tobytes() == w[..., ~mask].tobytes(), (t, k)      # the other robots are untouched
    # the masked robots solve on their first run after the reset, from the fresh state a period-1 tick with the same reset gives them
    for k in ("f_body", "status", "tau"):
        assert reset[t_r][k][..., mask].tobytes() == plain[t_r][k][..., mask].tobytes(), k
    assert any(reset[t_r][k][..., mask].tobytes() != walk[t_r][k][..., mask].tobytes() for k in ("f_body", "x0"))


@pytest.mark.parametrize("playback", [HOLD, PLAN], ids=["hold", "plan"])
def test_full_reset_repeats_the_first_runs(a1, engines, playback):
    eng = engines[10]
    B, T, t_r = 1024, 24, 12
    tp = _params(a1, a1.VARIANT_GAZEBO, "sched", 10)
    seqs, speed = tick_inputs(B, T, 51)
    # inputs from t_r on repeat the first ones, so that the reset tick sees what a fresh tick saw
    seqs = {k: np.ascontiguousarray(np.concatenate([v[:t_r], v[:T - t_r]])) for k, v in seqs.items()}
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        got = tick_run_rate(a1, eng, tp, ds, B, T, DT, [4] * T, playback, full_reset_at=t_r)
    finally:
        ds.free()
    assert first_difference(got[t_r:], got[:T - t_r]) is None


def test_host_arrays_match_device_arrays(a1, engines):
    eng = engines[10]
    B, T = 512, 12
    tp = _params(a1, a1.VARIANT_ISAAC, "sched", 10)
    seqs, speed = tick_inputs(B, T, 61)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        dev = tick_run_rate(a1, eng, tp, ds, B, T, DT, [3] * T, PLAN)
    finally:
        ds.free()
    tick = a1.Tick(eng, B, tp)
    try:
        tick.set_mpc_period(3, a1.PLAYBACK_PLAN)
        for t in range(T):
            tau, o = tick.run(DT, *(seqs[k][t] for k in a1.TICK_INPUTS[:-1]), speed)
            o["tau"] = tau
            for k in OUT_SPECS:
                assert o[k].tobytes() == dev[t][k].tobytes(), (t, k)
    finally:
        tick.close()


def test_argument_errors(a1, engines):
    eng = engines[10]
    B = 64
    tick = a1.Tick(eng, B, _params(a1, a1.VARIANT_GAZEBO, "held", 10))
    qp = a1.Tick(eng, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP))
    try:
        for period, pb, msg in ((0, PLAN, "period"), (11, PLAN, "period"), (-3, HOLD, "period"), (2, 2, "playback"), (2, -1, "playback")):
            with pytest.raises(a1.A1MpcError, match=msg):
                tick.set_mpc_period(period, pb)
        with pytest.raises(a1.A1MpcError, match="MPC mode"):
            qp.set_mpc_period(2, PLAN)
        tick.set_mpc_period(10, HOLD)
        tick.set_mpc_period(1, PLAN)
    finally:
        tick.close()
        qp.close()
    t20 = a1.Tick(engines[20], B, _params(a1, a1.VARIANT_GAZEBO, "held", 20))
    try:
        t20.set_mpc_period(20, PLAN)
        with pytest.raises(a1.A1MpcError, match="period"):
            t20.set_mpc_period(21, PLAN)
    finally:
        t20.close()
    L = a1.lib()
    z = np.zeros((12 * 10, 4))
    assert L.a1mpc_plan_forces_batch(eng.h, 0, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data) == -1


# ---- 3. against the oracle -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_against_oracle(a1, O, kind):
    D = tick_solve_inputs(512, 64, 43, 10)
    B, T, N, period = 512, 64, 10, 4
    tp = _params(a1, a1.VARIANT_GAZEBO, kind, N)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    tp.rho_opt[:], tp.rho_fix[:] = D["rho_opt"].tolist(), D["rho_fix"].tolist()
    tp.kp_foot[:], tp.kd_foot[:], tp.km_foot[:], tp.torques_gravity[:] = KP_ROS.tolist(), KD_ROS.tolist(), km.tolist(), tg.tolist()
    tp.use_terrain_adapt, tp.assume_flat_ground = 1, 1
    eng = a1.Engine(a1.default_config(horizon=N))
    ds = DeviceSeqs(a1, eng, D["seqs"], D["speed"])
    try:
        chain = staged_chain_rate(a1, eng, tp, ds, B, T, DT, [period] * T, PLAN, record=True)
        got = tick_run_rate(a1, eng, tp, ds, B, T, DT, [period] * T, PLAN)
    finally:
        ds.free()
        eng.close()
    assert first_difference(got, [{k: c[k] for k in OUT_SPECS} for c in chain]) is None
    # the due robots' QPs of every run
    sel = lambda k, t: chain[t][k][..., chain[t]["due"]]
    cat = lambda k: np.ascontiguousarray(np.concatenate([sel(k, t) for t in range(T)], axis=-1))
    st = dict(x0=cat("x0"), rot=cat("rot"), foot=cat("foot"), ref=cat("ref"), contact=cat("contacts"))
    f, status, iters = cat("f_body"), cat("status"), np.concatenate([chain[t]["iters"] for t in range(T)])
    cfg = O.make_config(horizon=N)
    if kind == "sched":
        fo, info = O.compute_grf_batch_ext(cfg, obatch(O, st), cat("sched"), None, O.MODE_EXACT, nthreads=O.hardware_threads())
    else:
        fo, info = O.compute_grf_batch(cfg, obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (info[:, 1] == 1).all()
    ef = np.abs(f - fo).max(axis=0)
    bad = np.nonzero((status != a1.STATUS_OPTIMAL) | ~(ef <= TOL_ORACLE))[0]
    counts = np.bincount(status, minlength=5).tolist()
    print("%s tick, period %d, %d due QPs of %d robot-runs: status counts %s, |f - f_oracle| max %.2e N, iterations median %d max %d" % (
        kind, period, f.shape[1], B * T, counts, float(ef.max()), int(np.median(iters)), int(iters.max())))
    assert bad.size == 0, "%d QPs fail (status %s, |f - f*| %s)" % (bad.size, status[bad][:8].tolist(), ef[bad][:8].tolist())
    assert f.shape[1] < 0.4 * B * T
