"""GPU tests of per-robot gaits in the control tick (a1mpc_tick_set_gaits).
  * Every output of every run of a tick with mixed gaits (robots cycling through trot, pace, bound, pronk, walk) bit-identical to the chain
    of staged entry points built with a1mpc_update_plan_gait_batch and a1mpc_swing_legs_gait_batch: the three adapter variants in QP mode,
    in the held MPC tick and in the scheduled MPC tick at B = 1024 over 40 stand / walk / stand runs, horizon 20, host = device rows and
    B = 65 536.
  * All-trot rows, and NULL after a gait, bit-identical to a tick that never called set_gaits.
  * What a pronk's flight phase gives: robots with no stance foot end A1MPC_STATUS_NO_CONTACT with zero forces (asserted for the held MPC
    tick, recorded for the others).
  * Argument errors leave the previous gaits in force.
  * Gaits with the other tick features, through their own tests' staged chains built on the gait entry points: ESTIMATED terrain and / or
    set_mpc_period(4), and a 25 % reset_robots mid-walk.  The chain's gait counters run by run: standstill holds the row's offsets (the
    start, a toggle to standstill and back mid-walk), walking advances each robot's own phase.
  * Against the oracle: every QP the staged gait chain poses on sched_tick_scenarios' closed loop (seed 43, B = 512 x 64 runs, N = 10),
    held and scheduled, solved again by the oracle's exact solve; per gait the status census, worst force error and stance-class mix."""
import ctypes as C

import numpy as np
import pytest

from command_scenarios import DT
from common import obatch
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, off, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)
TOL_LOOP = 1e-4     # N: the tolerance of the other closed-loop oracle tests (test_gpu_tick_sched.py)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def eng(a1):
    e = a1.Engine(a1.default_config(horizon=10))
    yield e
    e.close()


def mixed_rows(a1, B, shift=0):
    """robot b walks gait 1 + (b + shift) % 5 of a1mpc_gait_row, its four standstill offsets moved by 60 (b // 5 % 4) counts (mod cpg), so
    that within a short walk some robots of every gait reach the swing (a pronk its flight phase)"""
    rows = np.stack([a1.gait_row(1 + (b + shift) % 5) for b in range(B)], axis=1)
    rows[:4] = np.fmod(rows[:4] + 60.0 * ((np.arange(B) // 5) % 4)[None, :], rows[4][None, :])
    return np.ascontiguousarray(rows)


def long_inputs(B, T, seed):
    """tick_inputs with walking from run 5 to run 30 and standstill after it: stand / walk / stand"""
    seqs, speed = tick_inputs(B, min(T, 30), seed)
    if T > 30:
        rep = lambda a: np.ascontiguousarray(np.concatenate([a, np.repeat(a[-1:], T - 30, axis=0)]))
        seqs = {k: rep(v) for k, v in seqs.items()}
    seqs["cmd"][:, 6] = 0.0
    if T > 5:
        seqs["cmd"][5, 6] = 1.0
    if T > 30:
        seqs["cmd"][30, 6] = 1.0
    return seqs, speed


def staged_chain_gait(a1, eng, tp, ds, B, T, dt, d_gait, record=False):
    """the tick's stages as separate entry points on device pointers, with the two gait entry points in place of update_plan and the
    swing legs; QP mode, the held MPC tick (a1mpc_solve_batch_warm shift 0, cold at horizon 20) or the scheduled one (schedule row 0 = the
    swing stage's contacts, a1mpc_solve_batch_ext_warm shift 1, a1mpc_solve_batch_ext at horizon 20)"""
    L = a1.lib()
    mpc = tp.mode == a1.TICK_MPC
    N = eng.cfg.horizon
    sched = mpc and tp.gait.horizon != 0
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status")}
    d_sched = eng.dalloc(N * B * 4) if sched else None
    imu = eng.imu_alloc(B) if tp.command.variant != a1.VARIANT_HARDWARE else None
    sw, ekf = eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B))
    warm = eng.warm_alloc(B) if N == 10 and mpc else None
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), dv["ref"] if mpc else None, B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    inp = a1.Inputs(dv["x0"], dv["rot"], dv["foot"], dv["ref"], u["contact"], B)
    out = a1.Outputs(dv["f_body"], u["status"], None, None, B)
    ext = a1.InputsExt(d_sched.value, None) if sched else None
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    kdl, kpa, kda = arr(tp.kd_linear), arr(tp.kp_angular), arr(tp.kd_angular)
    res = []
    for t in range(T):
        a1._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                            dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                               rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, dt, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], dv["ref"] if mpc else None, B, dv["des"], B))
        lvd = off(dv["ref"], 5 * B * 8) if mpc else off(dv["des"], 6 * B * 8)
        a1._check(L.a1mpc_update_plan_gait_batch(eng.h, B, C.byref(tp.gait), d_gait, dv["gc"], ds.speed, u["mode"], x0p(9), lvd, dv["rz"], dv["rot"],
                                                 x0p(3), u["plan"], d_sched, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_gait_batch(eng.h, B, C.byref(tp.gait), d_gait, kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"],
                                                dv["rz"], dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        if sched:
            h2d(a1, eng, d_sched, d2h(a1, eng, u["contact"], B, np.uint32))
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                               ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        if mpc:
            a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
            if sched and warm is not None:
                a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out), warm, 1))
            elif sched:
                a1._check(L.a1mpc_solve_batch_ext(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out)))
            elif warm is not None:
                a1._check(L.a1mpc_solve_batch_warm(eng.h, B, C.byref(inp), C.byref(out), warm, 0))
            else:
                a1._check(L.a1mpc_solve_batch(eng.h, B, C.byref(inp), C.byref(out)))
        else:
            a1._check(L.a1mpc_stance_qp_batch(eng.h, B, C.c_size_t(B), dv["x0"], dv["rot"], dv["rz"], dv["foot"], u["contact"], dv["des"], dv["kpl"],
                                              kdl.ctypes.data, kpa.ctypes.data, kda.ctypes.data, dv["f_body"], u["status"], None))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        src = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"], ref=dv["ref"])
        res.append({k: d2h(a1, eng, src[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS if mpc or k != "ref"})
        if record:   # the gait counters, and the solve's inputs (ref after the terrain stage, the schedule with its row 0)
            res[-1].update(gc=d2h(a1, eng, dv["gc"], (4, B)), rot=d2h(a1, eng, dv["rot"], (9, B)), foot=d2h(a1, eng, dv["foot"], (12, B)),
                           ref_in=d2h(a1, eng, dv["ref"], (9, B)), sched=d2h(a1, eng, d_sched, (N, B), np.uint32) if sched else None)
    for p in list(dv.values()) + list(u.values()) + [d_sched, imu, sw, ekf, warm, cs]:
        if p is not None:
            L.a1mpc_device_free(eng.h, p)
    return res


def params(a1, variant, kind, N=10):
    tp = a1.default_tick_params(variant, a1.TICK_QP if kind == "qp" else a1.TICK_MPC)
    tp.gait.horizon = N if kind == "sched" else 0
    return tp


def run_tick(a1, eng, tp, ds, B, T, rows=None, host_rows=False, calls=None):
    tick = a1.Tick(eng, B, tp)
    try:
        for r in (calls or []):
            tick.set_gaits(r)
        if rows is not None:
            if host_rows:
                tick.set_gaits(rows)
            else:
                d = eng.dalloc(rows.nbytes)
                h2d(a1, eng, d, rows)
                tick.set_gaits_ptr(d.value)
                a1.lib().a1mpc_device_free(eng.h, d)   # the tick keeps its own copy
        return tick_run_device(a1, eng, tick, ds, B, T, DT)
    finally:
        tick.close()


def compare_with_chain(a1, eng, tp, B, T, seed, rows):
    seqs, speed = long_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    d = eng.dalloc(rows.nbytes)
    try:
        h2d(a1, eng, d, rows)
        want = staged_chain_gait(a1, eng, tp, ds, B, T, DT, d)
        got = run_tick(a1, eng, tp, ds, B, T, rows)
    finally:
        a1.lib().a1mpc_device_free(eng.h, d)
        ds.free()
    return got, want


def census(got, rows):
    """per gait: status counts over every run, and the stance-class mix of the contacts"""
    kinds = {1: "trot", 2: "pace", 3: "bound", 4: "pronk", 5: "walk"}
    out = {}
    for t, name in kinds.items():
        sel = np.arange(rows.shape[1]) % 5 == (t - 1)
        st = np.concatenate([g["status"][sel] for g in got])
        ns = np.concatenate([np.array([bin(int(c)).count("1") for c in g["contacts"][sel]]) for g in got])
        out[name] = dict(status=np.bincount(st, minlength=5).tolist(), stance=np.bincount(ns, minlength=5).tolist())
    return out


@pytest.mark.parametrize("kind", ["qp", "held", "sched"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_tick_with_mixed_gaits_bit_identical_to_staged_chain(a1, eng, variant, kind):
    B, T = 1024, 40
    rows = mixed_rows(a1, B)
    got, want = compare_with_chain(a1, eng, params(a1, VARIANTS[variant], kind), B, T, 81 + VARIANTS[variant], rows)
    assert first_difference(got, want) is None, first_difference(got, want)
    modes = np.array([g["movement_mode"] for g in got])
    assert modes[:5].sum() == 0 and modes[5:30].sum() > 0 and modes[-1].sum() == 0
    c = census(got, rows)
    print("%s %s: %s" % (variant, kind, c))
    # the pronk's flight phase: robots with no stance foot.  The held MPC tick answers them NO_CONTACT with zero forces; record what the
    # other ticks give them
    st = np.concatenate([g["status"] for g in got])
    ns = np.concatenate([g["contacts"] for g in got])
    fb = np.concatenate([g["f_body"] for g in got], axis=1)
    flight = ns == 0
    assert c["pronk"]["stance"][0] > 0 and flight.any()
    print("  flight robot-runs %d: status %s, max |f| %.3g" % (flight.sum(), np.bincount(st[flight], minlength=5).tolist(), np.abs(fb[:, flight]).max()))
    if kind == "held":
        assert (st[flight] == a1.STATUS_NO_CONTACT).all() and (fb[:, flight] == 0).all()


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_horizon_20(a1, kind):
    e = a1.Engine(a1.default_config(horizon=20))
    try:
        B, T = 512, 30
        got, want = compare_with_chain(a1, e, params(a1, 0, kind, N=20), B, T, 91, mixed_rows(a1, B, 2))
        assert first_difference(got, want) is None, first_difference(got, want)
    finally:
        e.close()


def test_large_batch(a1, eng):
    B, T = 65536, 4
    seqs, speed = long_inputs(B, T, 5)
    seqs["cmd"][:, 6] = 0.0
    seqs["cmd"][1, 6] = 1.0
    ds = DeviceSeqs(a1, eng, seqs, speed)
    rows = mixed_rows(a1, B)
    d = eng.dalloc(rows.nbytes)
    try:
        h2d(a1, eng, d, rows)
        tp = params(a1, 0, "sched")
        want = staged_chain_gait(a1, eng, tp, ds, B, T, DT, d)
        got = run_tick(a1, eng, tp, ds, B, T, rows)
    finally:
        a1.lib().a1mpc_device_free(eng.h, d)
        ds.free()
    assert first_difference(got, want) is None, first_difference(got, want)


@pytest.mark.parametrize("kind", ["qp", "held", "sched"])
def test_trot_rows_and_null_equal_the_plain_tick(a1, eng, kind):
    B, T = 1024, 40
    tp = params(a1, 0, kind)
    seqs, speed = long_inputs(B, T, 17)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        plain = run_tick(a1, eng, tp, ds, B, T)
        trot = run_tick(a1, eng, tp, ds, B, T, np.ascontiguousarray(np.repeat(a1.gait_row(a1.GAIT_TROT)[:, None], B, axis=1)))
        null_after = run_tick(a1, eng, tp, ds, B, T, calls=[mixed_rows(a1, B), None])
    finally:
        ds.free()
    assert first_difference(trot, plain) is None, first_difference(trot, plain)
    assert first_difference(null_after, plain) is None, first_difference(null_after, plain)


def test_host_rows_equal_device_rows(a1, eng):
    B, T = 512, 20
    tp = params(a1, 0, "sched")
    seqs, speed = long_inputs(B, T, 23)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    rows = mixed_rows(a1, B, 1)
    try:
        dev = run_tick(a1, eng, tp, ds, B, T, rows)
        host = run_tick(a1, eng, tp, ds, B, T, rows, host_rows=True)
    finally:
        ds.free()
    assert first_difference(host, dev) is None, first_difference(host, dev)


def test_argument_errors_keep_the_previous_gaits(a1, eng):
    B, T = 256, 20
    tp = params(a1, 0, "held")
    L = a1.lib()
    assert L.a1mpc_tick_set_gaits(None, None) == -1 and b"null argument" in L.a1mpc_last_error()
    with pytest.raises(a1.A1MpcError, match="unknown gait type"):
        a1.gait_row(9)
    rows = mixed_rows(a1, B)
    seqs, speed = long_inputs(B, T, 29)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        want = run_tick(a1, eng, tp, ds, B, T, rows)
        bad = []
        g = rows.copy(); g[3, 77] = np.nan; bad.append((g, "robot 77: a non-finite"))
        g = rows.copy(); g[5, 12] = g[4, 12]; bad.append((g, "robot 12: counter_per_swing"))
        g = rows.copy(); g[1, 200] = 240.0; bad.append((g, "robot 200: a reset offset"))
        g = rows.copy(); g[0, 5] = -1.0; bad.append((g, "robot 5: a reset offset"))
        tick = a1.Tick(eng, B, tp)
        try:
            tick.set_gaits(rows)
            for g, msg in bad:
                with pytest.raises(a1.A1MpcError, match=msg):
                    tick.set_gaits(g)
            with pytest.raises(ValueError):
                tick.set_gaits(rows[:, :10])
            got = tick_run_device(a1, eng, tick, ds, B, T, DT)
        finally:
            tick.close()
    finally:
        ds.free()
    assert first_difference(got, want) is None, first_difference(got, want)


# ---- gaits with the other tick features, through their own tests' chains -----------------------------------------------------------

class _GaitLib:
    """the library with a1mpc_update_plan_batch / a1mpc_swing_legs_batch answered by their gait entry points on d_gait: another test
    module's staged chain then is the chain of a tick with these gaits"""

    def __init__(self, L, d_gait):
        self._L, self._g = L, d_gait

    def __getattr__(self, name):
        return getattr(self._L, name)

    def a1mpc_update_plan_batch(self, h, B, gp, *rest):
        return self._L.a1mpc_update_plan_gait_batch(h, B, gp, self._g, *rest)

    def a1mpc_swing_legs_batch(self, h, B, gp, *rest):
        return self._L.a1mpc_swing_legs_gait_batch(h, B, gp, self._g, *rest)


class _GaitA1:
    """the a1mpc module as another test module's helpers use it, with every Tick given `rows` right after create and lib() = _GaitLib"""

    def __init__(self, a1, d_gait, rows):
        self._a1, self._lib, self._rows = a1, _GaitLib(a1.lib(), d_gait), rows

    def __getattr__(self, name):
        return getattr(self._a1, name)

    def lib(self):
        return self._lib

    def Tick(self, eng, B, tp):
        t = self._a1.Tick(eng, B, tp)
        t.set_gaits(self._rows)
        return t


@pytest.mark.parametrize("source,period", [("flat", 4), ("estimated", 1), ("estimated", 4)])
@pytest.mark.parametrize("kind", ["held", "sched"])
def test_gaits_with_terrain_and_mpc_period(a1, eng, kind, source, period):
    """the tick with mixed gaits, ESTIMATED terrain and / or set_mpc_period(4) (PLAYBACK_PLAN) against test_gpu_tick_rate.py's staged chain
    built on the gait entry points"""
    from test_gpu_tick_rate import ESTIMATED, FLAT, PLAN, staged_chain_rate, tick_run_rate
    B, T = 1024, 40
    tp = params(a1, 0, kind)
    rows = mixed_rows(a1, B)
    seqs, speed = long_inputs(B, T, 101)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    d = eng.dalloc(rows.nbytes)
    try:
        h2d(a1, eng, d, rows)
        A = _GaitA1(a1, d, rows)
        src = ESTIMATED if source == "estimated" else FLAT
        want = staged_chain_rate(A, eng, tp, ds, B, T, DT, [period] * T, PLAN, src)
        got = tick_run_rate(A, eng, tp, ds, B, T, DT, [period] * T, PLAN, src)
    finally:
        a1.lib().a1mpc_device_free(eng.h, d)
        ds.free()
    assert first_difference(got, want) is None, first_difference(got, want)


@pytest.mark.parametrize("kind", ["qp", "held", "sched"])
def test_reset_robots_mid_walk_with_gaits(a1, eng, kind):
    """a 25 % reset_robots mid-walk of a tick with mixed gaits (test_gpu_tick_reset.py's check): the masked robots continue exactly as the
    robots of a fresh tick with the same gaits created at the reset (which start in standstill on their rows' offsets), the others as the
    tick that saw no reset.  The gaits survive the reset"""
    from test_gpu_tick_reset import _check_resets, _diff
    B, T, R = 512, 74, 66
    rows = mixed_rows(a1, B)
    mask = (np.random.default_rng(77).random(B) < 0.25).astype(np.uint8)
    A = _GaitA1(a1, None, rows)
    got, want, untouched = _check_resets(A, eng, params(a1, 0, kind), B, T, {R: mask}, seed=45)
    assert _diff(got, want) is None, _diff(got, want)
    m = mask != 0
    assert any(not np.array_equal(got[t]["tau"][:, m], untouched[t]["tau"][:, m]) for t in range(R, T))


def test_counters_take_the_offsets_on_standstill_and_keep_their_phase_walking(a1, eng):
    """the gait counters of the chain that the tick reproduces bit for bit, run by run: a robot whose movement_mode is 0 (the start, a toggle
    to standstill and back mid-walk, the final stop) holds exactly its row's offsets; a walking robot advances its own phase,
    fmod(previous + speed, cpg).  A third of the robots toggle to standstill for one stretch mid-walk (cmd row 6)."""
    B, T = 1024, 40
    tp = params(a1, 0, "sched")
    rows = mixed_rows(a1, B, 3)
    seqs, speed = long_inputs(B, T, 111)
    tog = np.random.default_rng(8).random(B) < 1.0 / 3.0
    seqs["cmd"][15, 6, tog] = 1.0     # to standstill
    seqs["cmd"][17, 6, tog] = 1.0     # and back to walking
    ds = DeviceSeqs(a1, eng, seqs, speed)
    d = eng.dalloc(rows.nbytes)
    try:
        h2d(a1, eng, d, rows)
        want = staged_chain_gait(a1, eng, tp, ds, B, T, DT, d, record=True)
        got = run_tick(a1, eng, tp, ds, B, T, rows)
    finally:
        a1.lib().a1mpc_device_free(eng.h, d)
        ds.free()
    assert first_difference(got, [{k: w[k] for k in g} for g, w in zip(got, want)]) is None
    prev = np.zeros((4, B))
    stood_mid = np.zeros(B, bool)
    for t, w in enumerate(want):
        walk = w["movement_mode"] != 0
        assert np.array_equal(w["gc"][:, ~walk], rows[:4, ~walk]), t
        assert np.array_equal(w["gc"][:, walk], np.fmod(prev[:, walk] + speed[:, walk], rows[4][None, walk])), t
        if 10 <= t < 30:
            stood_mid |= ~walk
        prev = w["gc"]
    assert stood_mid[tog].any() and not stood_mid[~tog].any()
    print("robots toggled to standstill mid-walk: %d of %d" % (int(stood_mid.sum()), int(tog.sum())))
    assert (np.array([w["movement_mode"] for w in want])[-1] == 0).all()


# ---- against the oracle: every MPC QP the gait chain poses on the closed loop of sched_tick_scenarios -------------------------------

@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def closed_loop(built):
    from sched_tick_scenarios import tick_solve_inputs
    return tick_solve_inputs(512, 64, 43, 10)


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_mixed_gait_qps_against_the_oracle(a1, O, closed_loop, kind):
    """the raw inputs, leg geometry and gains of sched_tick_scenarios.tick_solve_inputs (seed 43, B = 512 x 64 runs, N = 10) through the
    staged gait chain with mixed gaits; every QP it poses (its x0, rot, foot, ref and contacts, on the scheduled tick its schedule) solved
    again by the oracle's exact solve: per gait the status census, the worst force error and the stance-class mix"""
    from swing_scenarios import KD_ROS, KP_ROS
    B, T, N = 512, 64, 10
    D = closed_loop
    tp = params(a1, a1.VARIANT_GAZEBO, kind, N)
    tp.rho_opt[:], tp.rho_fix[:] = D["rho_opt"].tolist(), D["rho_fix"].tolist()
    tp.kp_foot[:], tp.kd_foot[:] = KP_ROS.tolist(), KD_ROS.tolist()
    e = a1.Engine(a1.default_config(horizon=N))
    rows = mixed_rows(a1, B)
    ds = DeviceSeqs(a1, e, D["seqs"], D["speed"])
    d = e.dalloc(rows.nbytes)
    try:
        h2d(a1, e, d, rows)
        ch = staged_chain_gait(a1, e, tp, ds, B, T, DT, d, record=True)
    finally:
        a1.lib().a1mpc_device_free(e.h, d)
        ds.free()
        e.close()
    cat = lambda k: np.ascontiguousarray(np.concatenate([c[k] for c in ch], axis=-1))
    st = dict(x0=cat("x0"), rot=cat("rot"), foot=cat("foot"), ref=cat("ref_in"), contact=cat("contacts"))
    cfg = O.make_config(horizon=N)
    if kind == "sched":
        fo, info = O.compute_grf_batch_ext(cfg, obatch(O, st), cat("sched"), None, O.MODE_EXACT, nthreads=O.hardware_threads())
    else:
        fo, info = O.compute_grf_batch(cfg, obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    f, status = cat("f_body"), cat("status")
    gait = np.tile(np.arange(B) % 5, T)
    if kind == "sched":
        sch = cat("sched")
        anyc = np.bitwise_or.reduce(sch, axis=0)
        solved = anyc != 0
        mix = np.array([max(bin(int(x)).count("1") for x in col) for col in sch.T])
    else:
        solved = st["contact"] != 0
        mix = np.array([bin(int(x)).count("1") for x in st["contact"]])
    err = np.abs(f - fo).max(axis=0)
    lines = []
    for g, name in enumerate(("trot", "pace", "bound", "pronk", "walk")):
        sel = gait == g
        lines.append("%s: status %s, worst |f - f_oracle| %.2e N, stance classes %s" % (
            name, np.bincount(status[sel], minlength=5).tolist(), float(err[sel & solved].max()), np.bincount(mix[sel], minlength=5).tolist()))
    print("%s gait chain vs oracle (B = %d x %d runs): %d QPs\n  %s" % (kind, B, T, int(solved.sum()), "\n  ".join(lines)))
    assert (status[~solved] == a1.STATUS_NO_CONTACT).all() and (f[:, ~solved] == 0).all()
    assert (status[solved] == a1.STATUS_OPTIMAL).all(), np.bincount(status[solved], minlength=5)
    assert float(err[solved].max()) <= TOL_LOOP
