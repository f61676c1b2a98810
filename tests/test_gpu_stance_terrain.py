"""GPU tests of the QP-mode stance QP on terrain normals: a1mpc_stance_qp_batch_ext, a1mpc_surface_normals_batch and a QP-mode tick whose
stance pyramids stand on the walking surface (a1mpc_tick_set_stance_terrain).
  1. All-e_z normals, and normals = NULL, give f_body, status and root_acc bit-identical to a1mpc_stance_qp_batch (B = 16 384, all masks).
  2. Tilted per-foot normals at B = 65 536: every OPTIMAL robot within 1e-4 N of the exact solve of oracle/stance_terrain_oracle.cpp and
     inside its terrain pyramids to 1e-9 N; no IPM_ONLY or NUMERICAL; MAXITER (the 40-iteration cap) below 1e-4 of the stance robots.
  3. A NaN, Inf, zero or downward normal on a stance foot gives NUMERICAL and zero forces; the same on a swing foot changes nothing.
  4. Host arrays give what device arrays give, with ld > B.
  5. a1mpc_surface_normals_batch writes a1mpc_terrain_normals_batch's normals bit for bit and leaves the swing state bytewise untouched.
  6. Every output of every QP tick with ESTIMATED or GIVEN is bit-identical to the staged chain (the chain of tests/tick_scenarios.py with
     a1mpc_surface_normals_batch and a1mpc_stance_qp_batch_ext at stage 7): three variants at B = 1024 over 30 ticks, B = 65 536 for 3.
  7. FLAT, or never set, is the QP tick as it was; a 25 % reset_robots mid-walk and a full reset keep the source; FLAT -> ESTIMATED ->
     GIVEN -> FLAT mid-run matches the chain that switches alike; argument errors.
  8. The closed loop of the raw inputs of tests/sched_tick_scenarios.tick_solve_inputs (seed 43, B = 512 x 64 ticks) with ESTIMATED: the
     chain's own QPs against the oracle, and a census of the world-z solutions that would leave the terrain pyramid."""
import ctypes as C
import os

import numpy as np
import pytest

from command_scenarios import DT
from sched_tick_scenarios import _toggles
from stance_scenarios import gains, robots
from swing_scenarios import KD_RESET, KP_RESET, Scenario
from test_emu_stance_terrain import MAXITER, NUMERICAL, OPTIMAL, TOL_ORACLE, TOL_PYRAMID, check_against_oracle, ez_normals, pyramid_excess, tilted_normals
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, off, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)
FLAT, ESTIMATED, GIVEN = 0, 1, 2
QP_OUT = [k for k in OUT_SPECS if k != "ref"]
NTHREADS = os.cpu_count() or 1


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def OT(built):
    from oracle import stance_terrain_oracle_py
    return stance_terrain_oracle_py


@pytest.fixture(scope="module")
def engines(a1):
    es = {}

    def get(mass):
        if mass not in es:
            es[mass] = a1.Engine(a1.default_config(mass=mass))
        return es[mass]
    yield get
    for e in es.values():
        e.close()


def _args(st):
    return [st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")]


def _bits(a):
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def given_normals(B, T, seed):
    """[T][12][B] per-foot normals as a height-field lookup might give them: each foot its own, tilted up to 0.4 rad, changing every tick"""
    return np.stack([tilted_normals(B, seed + t, 0.4) for t in range(T)])


# ---- 1-4. the staged call ---------------------------------------------------------------------------------------------------------

def test_ez_and_null_normals_are_stance_qp_batch(a1, engines):
    B = 16384
    L = a1.lib()
    for y, name in enumerate(VARIANTS):
        mass, kdl, kpa, kda = gains(name)
        eng = engines(mass)
        st = robots(B, 60 + y, name, contact=np.arange(B) % 16)
        f0, s0, a0 = eng.stance_qp(*_args(st), kdl, kpa, kda, want_acc=True)
        f1, s1, a1_ = eng.stance_qp_ext(*_args(st), kdl, kpa, kda, ez_normals(B), want_acc=True)
        assert f1.tobytes() == f0.tobytes() and s1.tobytes() == s0.tobytes() and a1_.tobytes() == a0.tobytes(), name
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (st["x0"], st["rot"], st["rot_z"], st["foot"])]
        c = np.ascontiguousarray(st["contact"], dtype=np.uint32)
        g = [np.ascontiguousarray(v) for v in (st["des"], st["kp_linear"], kdl, kpa, kda)]
        f2, s2, a2 = np.zeros((12, B)), np.zeros(B, dtype=np.int32), np.zeros((6, B))
        a1._check(L.a1mpc_stance_qp_batch_ext(eng.h, B, B, *[v.ctypes.data for v in a], c.ctypes.data, *[v.ctypes.data for v in g], None,
                                              f2.ctypes.data, s2.ctypes.data, a2.ctypes.data))
        assert f2.tobytes() == f0.tobytes() and s2.tobytes() == s0.tobytes() and a2.tobytes() == a0.tobytes(), name
        print("%s: e_z and NULL normals bit-identical to a1mpc_stance_qp_batch; statuses %s" % (name, np.bincount(s0).tolist()))


def test_tilted_normals_against_the_oracle_65536(a1, OT, engines):
    B = 65536
    mass, kdl, kpa, kda = gains("gazebo")
    st = robots(B, 47, "gazebo")
    nrm = tilted_normals(B, 48)
    f, status, acc = engines(mass).stance_qp_ext(*_args(st), kdl, kpa, kda, nrm, want_acc=True)
    stance = (st["contact"] & 15) != 0
    ef, ep, nmax = check_against_oracle(OT, f, status, acc, st, nrm)
    assert nmax <= stance.sum() * 1e-4, nmax
    print("B=%d tilted normals: |f - f_oracle| %.2e N over %d OPTIMAL robots, pyramid excess %.2e N, MAXITER %d of %d stance robots"
          % (B, ef, int((status == OPTIMAL).sum()), ep, nmax, int(stance.sum())))


def test_invalid_normals(a1, engines):
    B = 4099
    mass, kdl, kpa, kda = gains("isaac")
    eng = engines(mass)
    st = robots(B, 71, "isaac", contact=np.full(B, 0b0111))
    nrm = tilted_normals(B, 72, 0.4)
    f0, s0 = eng.stance_qp_ext(*_args(st), kdl, kpa, kda, nrm)
    poison = [(np.nan, 0.0, 1.0), (0.0, np.inf, 1.0), (0.0, 0.0, -np.inf), (0.0, 0.0, 0.0), (0.3, 0.0, -0.9), (1.0, 0.0, 0.0), (0.0, 0.0, -1.0)]
    bad = nrm.copy()
    for i, v in enumerate(poison):
        bad[3 * (i % 3):3 * (i % 3) + 3, 4 * i] = v    # a stance foot
        bad[9:12, 4 * i + 1] = v                       # the swing foot
    f, s = eng.stance_qp_ext(*_args(st), kdl, kpa, kda, bad)
    hit = np.arange(len(poison)) * 4
    assert (s[hit] == NUMERICAL).all() and (f[:, hit] == 0.0).all()
    assert (s0[hit] != NUMERICAL).all()
    rest = np.setdiff1d(np.arange(B), hit)
    assert f[:, rest].tobytes() == f0[:, rest].tobytes() and s[rest].tobytes() == s0[rest].tobytes()


def test_host_and_device_arrays_agree_with_ld(a1, engines):
    B, ld = 3001, 3072
    L = a1.lib()
    mass, kdl, kpa, kda = gains("hardware")
    eng = engines(mass)
    st = robots(B, 81, "hardware")
    nrm = tilted_normals(B, 82)
    rows = dict(x0=12, rot=9, rot_z=9, foot=12, des=12, kp_linear=3, normals=12)
    data = dict(st, normals=nrm)
    wide = {k: np.zeros((r, ld)) for k, r in rows.items()}
    for k in rows:
        wide[k][:, :B] = data[k]
    c = np.ascontiguousarray(st["contact"], dtype=np.uint32)
    g = [np.ascontiguousarray(v) for v in (kdl, kpa, kda)]

    def call(ptr, f, s, acc):
        a1._check(L.a1mpc_stance_qp_batch_ext(eng.h, B, ld, ptr("x0"), ptr("rot"), ptr("rot_z"), ptr("foot"), ptr("contact"), ptr("des"),
                                              ptr("kp_linear"), *[v.ctypes.data for v in g], ptr("normals"), f, s, acc))
    fh, sh, ah = np.zeros((12, ld)), np.zeros(B, dtype=np.int32), np.zeros((6, ld))
    call(lambda k: c.ctypes.data if k == "contact" else wide[k].ctypes.data, fh.ctypes.data, sh.ctypes.data, ah.ctypes.data)
    d = {k: eng.dalloc(v.nbytes) for k, v in wide.items()}
    d["contact"] = eng.dalloc(c.nbytes)
    df, ds_, da = eng.dalloc(12 * ld * 8), eng.dalloc(B * 4), eng.dalloc(6 * ld * 8)
    try:
        for k, v in wide.items():
            h2d(a1, eng, d[k], v)
        h2d(a1, eng, d["contact"], c)
        call(lambda k: d[k], df, ds_, da)
        fd, sd, ad = d2h(a1, eng, df, (12, ld)), d2h(a1, eng, ds_, B, np.int32), d2h(a1, eng, da, (6, ld))
    finally:
        for p in list(d.values()) + [df, ds_, da]:
            L.a1mpc_device_free(eng.h, p)
    assert fh[:, :B].tobytes() == fd[:, :B].tobytes() and sh.tobytes() == sd.tobytes() and ah[:, :B].tobytes() == ad[:, :B].tobytes()
    f0, s0 = eng.stance_qp_ext(*_args(st), kdl, kpa, kda, nrm)
    assert fh[:, :B].tobytes() == f0.tobytes() and sh.tobytes() == s0.tobytes()
    assert (sh[(st["contact"] & 15) != 0] == OPTIMAL).mean() > 0.999


# ---- 5. the staged normals --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("host", [True, False], ids=["host", "device"])
def test_surface_normals_batch_matches_terrain_normals_batch(a1, engines, host):
    eng = engines(12.0)
    L = a1.lib()
    B, T = 1024, 160
    sc = Scenario(B, 17)
    gp = a1.default_gait_params()
    s0, s1 = eng.swing_alloc(B), eng.swing_alloc(B)
    nbytes = L.a1mpc_swing_bytes(B)
    dpos, dnrm = eng.dalloc(3 * B * 8), eng.dalloc(12 * B * 8)
    tilted = 0
    try:
        for t in range(T):
            x = sc.tick()
            args = (x["gait_counter"], x["plan_contacts"], x["rot_z"], x["foot_pos_abs"], x["foot_pos_target_rel"], x["foot_force"])
            eng.swing_legs(gp, KP_RESET, KD_RESET, s0, DT, *args)
            eng.swing_legs(gp, KP_RESET, KD_RESET, s1, DT, *args)
            before = d2h(a1, eng, s0, nbytes // 8)
            if host:
                nrm = eng.surface_normals(s0, x["root_pos"])
            else:
                h2d(a1, eng, dpos, x["root_pos"])
                a1._check(L.a1mpc_surface_normals_batch(eng.h, B, s0, dpos, dnrm))
                nrm = d2h(a1, eng, dnrm, (12, B))
            assert d2h(a1, eng, s0, nbytes // 8).tobytes() == before.tobytes(), t
            _, want = eng.terrain_normals(s1, 1, x["root_pos"], np.zeros((9, B)))   # advances s1's filter: a copy of the recent contacts
            assert nrm.tobytes() == want.tobytes(), t
            tilted += int((nrm[2] < 1.0 - 1e-6).sum())
    finally:
        for p in (s0, s1, dpos, dnrm):
            L.a1mpc_device_free(eng.h, p)
    print("surface_normals (%s arrays): %d ticks bit-identical to terrain_normals, %d tilted robot-ticks" % ("host" if host else "device", T, tilted))
    assert tilted > 0


# ---- 6-8. the tick ----------------------------------------------------------------------------------------------------------------

def staged_chain_stance(a1, eng, tp, ds, B, T, dt, sources, given=None, record=False):
    """the QP-mode tick's stages as separate entry points on device pointers, from the same start state as a1mpc_tick_create: the chain of
    tests/tick_scenarios.staged_chain, and at stage 7 per sources[t] a1mpc_stance_qp_batch (FLAT) or a1mpc_stance_qp_batch_ext with the
    normals of a1mpc_surface_normals_batch (ESTIMATED) or given[t] [12][B] (GIVEN).  One dict of host outputs per tick; with record, also
    the QP's data (root_acc, rot_z, rot, foot, normals)."""
    L = a1.lib()
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, gc=4, trel=12, fk=12, f_body=12, tau=12, nrm=12,
              acc=6)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status")}
    imu = eng.imu_alloc(B) if tp.command.variant != a1.VARIANT_HARDWARE else None
    sw, ekf = eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B))
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), None, B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    kdl, kpa, kda = arr(tp.kd_linear), arr(tp.kp_angular), arr(tp.kd_angular)
    res = []
    try:
        for t in range(T):
            a1._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                                dv["ia"], dv["ig"]))
            a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                                   rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
            a1._check(L.a1mpc_command_batch(eng.h, B, cs, dt, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], None, B, dv["des"], B))
            a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(tp.gait), dv["gc"], ds.speed, u["mode"], x0p(9), off(dv["des"], 6 * B * 8), dv["rz"],
                                                dv["rot"], x0p(3), u["plan"], None, dv["trel"], None, None))
            a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"], dv["rz"],
                                               dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
            if t == 0:
                a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
            else:
                a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"],
                                                   dv["fvr"], ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
            qp = (eng.h, B, C.c_size_t(B), dv["x0"], dv["rot"], dv["rz"], dv["foot"], u["contact"], dv["des"], dv["kpl"], kdl.ctypes.data,
                  kpa.ctypes.data, kda.ctypes.data)
            src = sources[t]
            if src == FLAT:
                a1._check(L.a1mpc_stance_qp_batch(*qp, dv["f_body"], u["status"], dv["acc"]))
            else:
                if src == ESTIMATED:
                    a1._check(L.a1mpc_surface_normals_batch(eng.h, B, sw, x0p(3), dv["nrm"]))
                else:
                    h2d(a1, eng, dv["nrm"], given[t])
                a1._check(L.a1mpc_stance_qp_batch_ext(*qp, dv["nrm"], dv["f_body"], u["status"], dv["acc"]))
            a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
            srcs = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"])
            r = {k: d2h(a1, eng, srcs[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in QP_OUT}
            if record:
                r.update(root_acc=d2h(a1, eng, dv["acc"], (6, B)), rot_z=d2h(a1, eng, dv["rz"], (9, B)), rot=d2h(a1, eng, dv["rot"], (9, B)),
                         foot=d2h(a1, eng, dv["foot"], (12, B)), normals=d2h(a1, eng, dv["nrm"], (12, B)) if src != FLAT else None)
            res.append(r)
    finally:
        for p in list(dv.values()) + list(u.values()) + [imu, sw, ekf, cs]:
            if p is not None:
                L.a1mpc_device_free(eng.h, p)
    return res


def tick_run_stance(a1, eng, tp, ds, B, T, dt, sources, given=None, resets=None, full_reset=None, t0=0):
    """ticks t0 .. T-1 of a fresh QP tick on device pointers; set_stance_terrain(sources[t]) before tick t whenever the source changes (GIVEN
    binds one device buffer, given[t] is written into it before the run); resets {t: mask}: reset_robots_ptr before tick t; full_reset: the
    tick before which a1mpc_tick_reset runs.  One dict per tick."""
    L = a1.lib()
    d = {k: eng.dalloc(int(np.prod(OUT_SPECS[k][0] + (B,))) * np.dtype(OUT_SPECS[k][1]).itemsize) for k in QP_OUT}
    outs = a1.TickOutputs(*[d.get(k) for k in a1.TICK_OUTPUTS])
    d_given, d_mask = eng.dalloc(12 * B * 8), eng.dalloc(B)
    tick = a1.Tick(eng, B, tp)
    res, cur = [], FLAT
    try:
        for t in range(t0, T):
            if sources[t] != cur:
                tick.set_stance_terrain(sources[t], d_given.value if sources[t] == GIVEN else 0)
                cur = sources[t]
            if cur == GIVEN:
                h2d(a1, eng, d_given, given[t])
            if resets and t in resets:
                h2d(a1, eng, d_mask, np.ascontiguousarray(resets[t], dtype=np.uint8))
                tick.reset_robots_ptr(d_mask.value)
            if full_reset == t:
                tick.reset()
            ins = a1.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1.TICK_INPUTS])
            tick.run_ptrs(dt, ins, outs)
            res.append({k: d2h(a1, eng, d[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in QP_OUT})
    finally:
        tick.close()
        for p in list(d.values()) + [d_given, d_mask]:
            L.a1mpc_device_free(eng.h, p)
    return res


def _qp_params(a1, variant):
    return a1.default_tick_params(variant, a1.TICK_QP)


def _compare(a1, eng, tp, B, T, seed, sources):
    seqs, speed = tick_inputs(B, T, seed)
    given = given_normals(B, T, seed + 100) if GIVEN in sources else None
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        want = staged_chain_stance(a1, eng, tp, ds, B, T, DT, sources, given)
        got = tick_run_stance(a1, eng, tp, ds, B, T, DT, sources, given)
    finally:
        ds.free()
    return got, want


@pytest.mark.parametrize("source", [ESTIMATED, GIVEN], ids=["estimated", "given"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_tick_bit_identical_to_staged_chain(a1, engines, variant, source):
    B, T = 1024, 30
    got, want = _compare(a1, engines(12.0), _qp_params(a1, VARIANTS[variant]), B, T, 11 + VARIANTS[variant], [source] * T)
    assert first_difference(got, want) is None, first_difference(got, want)
    print("%s %s: %d ticks bit-identical; statuses of the last tick %s" % (variant, "ESTIMATED" if source == ESTIMATED else "GIVEN", T,
                                                                         np.bincount(got[-1]["status"], minlength=5).tolist()))


@pytest.mark.parametrize("source", [ESTIMATED, GIVEN], ids=["estimated", "given"])
def test_large_batch_bit_identical(a1, engines, source):
    got, want = _compare(a1, engines(12.0), _qp_params(a1, a1.VARIANT_GAZEBO), 65536, 3, 13, [source] * 3)
    assert first_difference(got, want) is None, first_difference(got, want)


def test_flat_is_the_qp_tick_as_it_was(a1, engines):
    eng = engines(12.0)
    B, T = 1024, 30
    tp = _qp_params(a1, a1.VARIANT_GAZEBO)
    seqs, speed = tick_inputs(B, T, 21)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    runs = {}
    try:
        for how in ("never", "flat", "estimated_then_flat"):
            tick = a1.Tick(eng, B, tp)
            try:
                if how == "flat":
                    tick.set_stance_terrain(a1.TERRAIN_FLAT)
                elif how == "estimated_then_flat":
                    tick.set_stance_terrain(a1.TERRAIN_ESTIMATED)
                    tick.set_stance_terrain(a1.TERRAIN_FLAT)
                runs[how] = tick_run_device(a1, eng, tick, ds, B, T, DT)
            finally:
                tick.close()
        chain = staged_chain_stance(a1, eng, tp, ds, B, T, DT, [FLAT] * T)
        est = tick_run_stance(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T)
    finally:
        ds.free()
    assert first_difference(chain, runs["never"]) is None
    for how in ("flat", "estimated_then_flat"):
        assert first_difference(runs[how], runs["never"]) is None, (how, first_difference(runs[how], runs["never"]))
    # stage 7 writes nothing but the forces: the state the next tick starts from does not depend on them within a tick
    assert all(np.array_equal(e["contacts"], w["contacts"]) and np.array_equal(e["movement_mode"], w["movement_mode"]) for e, w in zip(est, runs["never"]))


def test_reset_keeps_the_source(a1, engines):
    eng = engines(12.0)
    B, T, tr = 1024, 30, 14
    tp = _qp_params(a1, a1.VARIANT_HARDWARE)
    seqs, speed = tick_inputs(B, T, 31)
    mask = np.random.default_rng(32).random(B) < 0.25
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        src = [ESTIMATED] * T
        a = tick_run_stance(a1, eng, tp, ds, B, T, DT, src, resets={tr: mask})
        u = tick_run_stance(a1, eng, tp, ds, B, T, DT, src)
        f = tick_run_stance(a1, eng, tp, ds, B, T, DT, src, t0=tr)
        full = tick_run_stance(a1, eng, tp, ds, B, T, DT, src, full_reset=tr)
    finally:
        ds.free()
    assert first_difference(a[:tr], u[:tr]) is None
    for t in range(tr, T):
        for k in QP_OUT:
            assert a[t][k][..., mask].tobytes() == f[t - tr][k][..., mask].tobytes(), (t, k, "reset robots")
            assert a[t][k][..., ~mask].tobytes() == u[t][k][..., ~mask].tobytes(), (t, k, "other robots")
    assert first_difference(full[:tr], u[:tr]) is None and first_difference(full[tr:], f) is None


def test_switching_source_mid_run(a1, engines):
    B, T = 1024, 30
    sources = [FLAT] * 6 + [ESTIMATED] * 8 + [GIVEN] * 6 + [FLAT] * 4 + [ESTIMATED] * 6
    got, want = _compare(a1, engines(12.0), _qp_params(a1, a1.VARIANT_ISAAC), B, T, 41, sources)
    assert first_difference(got, want) is None, first_difference(got, want)


def test_argument_errors(a1, engines):
    L = a1.lib()
    eng = engines(12.0)
    B = 64
    buf = np.zeros((12, B))
    d_nrm = eng.dalloc(12 * B * 8)
    qp = a1.Tick(eng, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP))
    mpc = a1.Tick(eng, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC))
    sw = eng.swing_alloc(B)
    try:
        err = lambda: L.a1mpc_last_error()
        assert L.a1mpc_tick_set_stance_terrain(None, ESTIMATED, None) == -1 and b"null argument" in err()
        for s in (FLAT, ESTIMATED, GIVEN):
            assert L.a1mpc_tick_set_stance_terrain(mpc.t, s, d_nrm) == -1 and b"a1mpc_tick_set_terrain" in err()
        for s in (-1, 3, 100):
            assert L.a1mpc_tick_set_stance_terrain(qp.t, s, None) == -1 and b"unknown terrain source" in err()
        assert L.a1mpc_tick_set_stance_terrain(qp.t, GIVEN, None) == -1 and b"needs a normals array" in err()
        assert L.a1mpc_tick_set_stance_terrain(qp.t, GIVEN, buf.ctypes.data) == -1 and b"device memory" in err()
        assert L.a1mpc_tick_set_terrain(qp.t, ESTIMATED, None) == -1 and b"MPC mode" in err()    # the MPC call's contract is unchanged
        assert L.a1mpc_tick_set_stance_terrain(qp.t, GIVEN, d_nrm) == 0 and L.a1mpc_tick_set_stance_terrain(qp.t, ESTIMATED, d_nrm) == 0
        assert L.a1mpc_tick_set_stance_terrain(qp.t, FLAT, None) == 0
        P = lambda a: a.ctypes.data
        pos = np.full((3, B), 0.3)
        assert L.a1mpc_surface_normals_batch(eng.h, B, sw, P(pos), None) == -1 and b"null argument" in err()
        assert L.a1mpc_surface_normals_batch(eng.h, B, sw, None, P(buf)) == -1
        assert L.a1mpc_surface_normals_batch(eng.h, 0, sw, P(pos), P(buf)) == -1
        assert L.a1mpc_surface_normals_batch(eng.h, B, P(buf), P(pos), P(buf)) == -1 and b"device memory" in err()
        assert L.a1mpc_surface_normals_batch(eng.h, B, sw, P(pos), d_nrm) == -1 and b"all-host or all-device" in err()
        assert L.a1mpc_surface_normals_batch(eng.h, B, sw, P(pos), P(buf)) == 0 and (buf[2::3] == 1.0).all() and (buf[0::3] == 0.0).all()
        st = robots(B, 3, "gazebo")
        a = [np.ascontiguousarray(st[k]) for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")]
        g = [np.ascontiguousarray(v) for v in gains("gazebo")[1:]]
        f, s = np.zeros((12, B)), np.zeros(B, dtype=np.int32)
        assert L.a1mpc_stance_qp_batch_ext(eng.h, B, B - 1, *[P(v) for v in a], *[P(v) for v in g], P(buf), P(f), P(s), None) == -1
        assert L.a1mpc_stance_qp_batch_ext(eng.h, B, B, *[P(v) for v in a], *[P(v) for v in g], d_nrm, P(f), P(s), None) == -1
        seqs, speed = tick_inputs(B, 2, 9)
        tau, o = qp.run(DT, *(seqs[n][0] for n in a1.TICK_INPUTS[:-1]), speed)
        assert np.isfinite(tau).all() and (o["status"] == a1.STATUS_OPTIMAL).all()
    finally:
        for tk in (qp, mpc):
            tk.close()
        L.a1mpc_device_free(eng.h, d_nrm)
        L.a1mpc_device_free(eng.h, sw)


def test_closed_loop_against_the_oracle(a1, OT, engines):
    """the raw inputs of sched_tick_scenarios.tick_solve_inputs (seed 43): tick_inputs with its contact toggles, B = 512 x 64 ticks"""
    eng = engines(12.0)
    B, T = 512, 64
    seqs, speed = tick_inputs(B, T, 43)
    seqs["cmd"][:, 6] = _toggles(B, T)
    seqs["cmd"] = np.ascontiguousarray(seqs["cmd"])
    tp = _qp_params(a1, a1.VARIANT_GAZEBO)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        chain = staged_chain_stance(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T, record=True)
        got = tick_run_stance(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T)
    finally:
        ds.free()
    assert first_difference(got, [{k: c[k] for k in QP_OUT} for c in chain]) is None
    cat = lambda k: np.concatenate([c[k] for c in chain], axis=-1)
    f, status, acc, rz, rot, foot, con, nrm = (cat(k) for k in ("f_body", "status", "root_acc", "rot_z", "rot", "foot", "contacts", "normals"))
    st = dict(rot_z=rz, rot=rot, foot=foot, contact=con)
    stance = (con & 15) != 0
    ef, ep, nmax = check_against_oracle(OT, f, status, acc, st, nrm)
    assert nmax <= stance.sum() * 1e-4, nmax
    fz, _ = OT.grf_qp_batch_ext(acc, rz, rot, foot, con, np.tile(np.array([0.0, 0.0, 1.0]), 4)[:, None].repeat(con.size, axis=1), NTHREADS)
    ex = pyramid_excess(fz[:, stance], rot[:, stance], con[stance], nrm[:, stance])
    tilt = np.arccos(np.clip(nrm[2, stance], -1.0, 1.0))
    print("closed loop B=%d x %d ticks, ESTIMATED: %d stance robot-ticks, statuses %s; |f - f_oracle| %.2e N, pyramid excess %.2e N, MAXITER %d; "
          "world-z solutions outside the terrain pyramid: %d (%d by more than 1 N, worst %.2f N); tilt median %.4f rad, max %.4f rad"
          % (B, T, int(stance.sum()), np.bincount(status, minlength=5).tolist(), ef, ep, nmax, int((ex > TOL_PYRAMID).sum()), int((ex > 1.0).sum()),
             float(ex.max()), float(np.median(tilt)), float(tilt.max())))
