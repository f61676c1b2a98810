"""GPU tests of a tick whose MPC friction pyramids stand on the walking surface (a1mpc_tick_set_terrain) and of its staged entry point
a1mpc_terrain_normals_batch.
  1. a1mpc_terrain_normals_batch writes, bit for bit, what a1mpc_terrain_pitch_batch writes (ref row 1, terrain_pitch, the swing state),
     and normals within 1e-13 of the numpy restatement of tests/test_emu_terrain_normals.py.
  2. Every output of every tick is bit-identical to the hand-built chain of staged entry points (staged_chain_terrain below: the chain of
     tests/tick_scenarios.py, or of test_gpu_tick_sched.py for the scheduled tick, with a1mpc_terrain_normals_batch at stage 7 and then
     a1mpc_solve_batch_ext_warm / a1mpc_solve_batch_ext with those normals, or the given ones; the held pattern as the swing stage's
     contacts repeated over N rows): three variants x {held, scheduled} x N = 10, 20 x {ESTIMATED, GIVEN} at B = 1024 over 30 ticks,
     B = 65 536 for 3 ticks, on the default handle and on an A1MPC_EXT_COMPACT=0 handle.
  3. Against the oracle, on the closed loop of tests/sched_tick_scenarios.tick_solve_inputs (seed 43, B = 512 x 64 ticks): the chain's
     own QPs and normals, every QP OPTIMAL and within 1e-4 N of compute_grf_batch_ext; every stance force inside its foot's terrain
     pyramid to 1e-6 N; and a census of the robots whose world-z solution would have left that pyramid.
  4. FLAT, never set or set back, is bit-identical to a tick that never heard of terrain; where the estimated normal is exactly e_z,
     ESTIMATED agrees with FLAT to 1e-8 N.
  5. Terrain and reset: reset_robots on 25 % mid-walk gives a fresh terrain tick for those robots and the untouched run for the rest, bit
     for bit; a1mpc_tick_reset reproduces the first ticks; FLAT -> ESTIMATED -> FLAT mid-run matches the chain that switches alike.
  6. Argument errors."""
import ctypes as C
import os

import numpy as np
import pytest

from command_scenarios import DT
from common import obatch
from sched_tick_scenarios import tick_solve_inputs
from swing_scenarios import KD_RESET, KD_ROS, KP_RESET, KP_ROS, Scenario
from test_emu_terrain_normals import restated_normals
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, off, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)
FLAT, ESTIMATED, GIVEN = 0, 1, 2
TOL_ORACLE = 1e-4   # N: the tolerance of the scheduled tick against the oracle (test_gpu_tick_sched.py)
TOL_PYRAMID = 1e-6  # N


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def _engine(a1, horizon=10, compact=True, **kw):
    if compact:
        return a1.Engine(a1.default_config(horizon=horizon, **kw))
    os.environ["A1MPC_EXT_COMPACT"] = "0"
    try:
        return a1.Engine(a1.default_config(horizon=horizon, **kw))
    finally:
        del os.environ["A1MPC_EXT_COMPACT"]


@pytest.fixture(scope="module")
def engines(a1):
    es = {"10": _engine(a1, 10), "10_general": _engine(a1, 10, compact=False), "20": _engine(a1, 20)}
    yield es
    for e in es.values():
        e.close()


def _params(a1, variant, kind, N):
    """kind: held (gait.horizon 0) or sched (gait.horizon N), MPC mode"""
    tp = a1.default_tick_params(variant, a1.TICK_MPC)
    if kind == "sched":
        tp.gait.horizon = N
    return tp


def given_normals(B, T, seed):
    """[T][12][B] per-foot normals as a height-field lookup might give them: each foot its own, tilted up to 0.3 rad, changing every tick"""
    rng = np.random.default_rng(seed)
    tilt, az = rng.uniform(0.0, 0.3, (T, 4, B)), rng.uniform(-np.pi, np.pi, (T, 4, B))
    n = np.stack([np.sin(tilt) * np.cos(az), np.sin(tilt) * np.sin(az), np.cos(tilt)], axis=2)   # [T,4,3,B]
    return np.ascontiguousarray(n.reshape(T, 12, B))


def staged_chain_terrain(a1, eng, tp, ds, B, T, dt, sources, given=None, record=False):
    """the tick's stages as separate entry points on device pointers (MPC mode), from the same start state as a1mpc_tick_create.  sources[t]:
    FLAT (a1mpc_terrain_pitch_batch and the tick's world-z solve) or ESTIMATED / GIVEN (a1mpc_terrain_normals_batch, then the _ext solve with
    its normals or with given[t] [12][B]: on the held pattern, the swing stage's contacts in all N rows, warm with shift 0; on the schedule
    of the scheduled tick, warm with shift 1; cold at horizon 20).  The schedule's rows are copied through the host: the C ABI has no
    device-to-device copy.  One dict of host outputs per tick; with record, also the solve's inputs (x0, rot, foot, ref, sched, normals)."""
    L = a1.lib()
    N = eng.cfg.horizon
    sched_tick = tp.gait.horizon == N
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12,
              nrm=12, given=12)
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
                                            dv["rot"], x0p(3), u["plan"], d_sched if sched_tick else None, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"], dv["rz"],
                                           dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        src = sources[t]
        con = d2h(a1, eng, u["contact"], B, np.uint32)
        if sched_tick:
            h2d(a1, eng, d_sched, con)                                           # row 0 of the schedule
        elif src != FLAT:
            h2d(a1, eng, d_sched, np.tile(con, (N, 1)))                          # the held pattern over the horizon
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                               ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        if src == FLAT:
            a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
            nrm = None
        else:
            a1._check(L.a1mpc_terrain_normals_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None, dv["nrm"]))
            if src == GIVEN:
                h2d(a1, eng, dv["given"], given[t])
            nrm = dv["nrm"] if src == ESTIMATED else dv["given"]
        ext = a1.InputsExt(d_sched.value, nrm.value if nrm is not None else None)
        shift = 1 if sched_tick else 0
        if src == FLAT and not sched_tick:
            if warm is not None:
                a1._check(L.a1mpc_solve_batch_warm(eng.h, B, C.byref(inp), C.byref(out), warm, 0))
            else:
                a1._check(L.a1mpc_solve_batch(eng.h, B, C.byref(inp), C.byref(out)))
        elif warm is not None:
            a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out), warm, shift))
        else:
            a1._check(L.a1mpc_solve_batch_ext(eng.h, B, C.byref(inp), C.byref(ext), C.byref(out)))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        srcs = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"], ref=dv["ref"])
        r = {k: d2h(a1, eng, srcs[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS}
        if record:
            r.update(rot=d2h(a1, eng, dv["rot"], (9, B)), foot=d2h(a1, eng, dv["foot"], (12, B)),
                     sched=d2h(a1, eng, d_sched, (N, B), np.uint32) if (sched_tick or src != FLAT) else np.tile(con, (N, 1)),
                     normals=d2h(a1, eng, nrm, (12, B)) if nrm is not None else None)
        res.append(r)
    for p in list(dv.values()) + list(u.values()) + [d_sched, imu, sw, ekf, warm, cs]:
        if p is not None:
            L.a1mpc_device_free(eng.h, p)
    return res


def tick_run_terrain(a1, eng, tp, ds, B, T, dt, sources, given=None, resets=None, t0=0):
    """ticks t0 .. T-1 of a fresh tick on device pointers; set_terrain(sources[t]) before tick t whenever the source changes (GIVEN binds one
    device buffer, given[t] is written into it before the run); resets {t: mask}: reset_robots_ptr before tick t.  One dict per tick."""
    L = a1.lib()
    d = {k: eng.dalloc(int(np.prod(OUT_SPECS[k][0] + (B,))) * np.dtype(OUT_SPECS[k][1]).itemsize) for k in OUT_SPECS}
    outs = a1.TickOutputs(*[d.get(k) for k in a1.TICK_OUTPUTS])
    d_given, d_mask = eng.dalloc(12 * B * 8), eng.dalloc(B)
    tick = a1.Tick(eng, B, tp)
    res, cur = [], FLAT
    try:
        for t in range(t0, T):
            if sources[t] != cur:
                tick.set_terrain(sources[t], d_given.value if sources[t] == GIVEN else 0)
                cur = sources[t]
            if cur == GIVEN:
                h2d(a1, eng, d_given, given[t])
            if resets and t in resets:
                h2d(a1, eng, d_mask, np.ascontiguousarray(resets[t], dtype=np.uint8))
                tick.reset_robots_ptr(d_mask.value)
            ins = a1.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1.TICK_INPUTS])
            tick.run_ptrs(dt, ins, outs)
            res.append({k: d2h(a1, eng, d[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS})
    finally:
        tick.close()
        for p in list(d.values()) + [d_given, d_mask]:
            L.a1mpc_device_free(eng.h, p)
    return res


def _compare(a1, eng, tp, B, T, seed, sources):
    seqs, speed = tick_inputs(B, T, seed)
    given = given_normals(B, T, seed + 100) if GIVEN in sources else None
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        want = staged_chain_terrain(a1, eng, tp, ds, B, T, DT, sources, given)
        got = tick_run_terrain(a1, eng, tp, ds, B, T, DT, sources, given)
    finally:
        ds.free()
    return got, want


def _status_counts(got):
    return [np.bincount(g["status"], minlength=5).tolist() for g in got]


# ---- 1. the staged entry point against a1mpc_terrain_pitch_batch -------------------------------------------------------------------

@pytest.mark.parametrize("host", [True, False], ids=["host", "device"])
def test_terrain_normals_batch_matches_terrain_pitch_batch(a1, engines, host):
    eng = engines["10"]
    L = a1.lib()
    B, T = 1024, 160
    sc = Scenario(B, 17)
    gp = a1.default_gait_params()
    s0, s1 = eng.swing_alloc(B), eng.swing_alloc(B)
    nbytes = L.a1mpc_swing_bytes(B)
    dref, dpos, dpitch, dnrm = eng.dalloc(9 * B * 8), eng.dalloc(3 * B * 8), eng.dalloc(B * 8), eng.dalloc(12 * B * 8)
    worst, compared, tilted = 0.0, 0, 0
    try:
        for t in range(T):
            x = sc.tick()
            args = (x["gait_counter"], x["plan_contacts"], x["rot_z"], x["foot_pos_abs"], x["foot_pos_target_rel"], x["foot_force"])
            _, _, _, rc = eng.swing_legs(gp, KP_RESET, KD_RESET, s0, DT, *args)
            eng.swing_legs(gp, KP_RESET, KD_RESET, s1, DT, *args)
            ref0, ref1 = np.full((9, B), 3.0), np.full((9, B), 3.0)
            p0 = eng.terrain_pitch(s0, 1, x["root_pos"], ref0)
            if host:
                p1, nrm = eng.terrain_normals(s1, 1, x["root_pos"], ref1)
            else:
                h2d(a1, eng, dref, ref1)
                h2d(a1, eng, dpos, x["root_pos"])
                a1._check(L.a1mpc_terrain_normals_batch(eng.h, B, s1, 1, dpos, dref, B, dpitch, dnrm))
                ref1, p1, nrm = d2h(a1, eng, dref, (9, B)), d2h(a1, eng, dpitch, B), d2h(a1, eng, dnrm, (12, B))
            assert ref1.tobytes() == ref0.tobytes() and p1.tobytes() == p0.tobytes(), t
            assert d2h(a1, eng, s1, nbytes // 8).tobytes() == d2h(a1, eng, s0, nbytes // 8).tobytes(), t
            assert np.array_equal(nrm, np.tile(nrm[0:3], (4, 1))) and (nrm[2] > 0.0).all()
            want, margin = restated_normals(rc, x["root_pos"][2])
            ok = margin > 1e6
            worst = max(worst, float(np.abs(nrm[0:3, ok] - want[:, ok]).max())) if ok.any() else worst
            compared += int(ok.sum())
            tilted += int((nrm[2] < 1.0 - 1e-6).sum())
    finally:
        for p in (s0, s1, dref, dpos, dpitch, dnrm):
            L.a1mpc_device_free(eng.h, p)
    print("terrain_normals vs terrain_pitch (%s arrays): %d ticks bit-identical; normals vs numpy %.2e over %d robot-ticks, %d tilted" % (
        "host" if host else "device", T, worst, compared, tilted))
    assert worst <= 1e-13 and compared >= 0.9 * B * T and tilted > 0


# ---- 2. the tick against the staged chain ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("source", [ESTIMATED, GIVEN], ids=["estimated", "given"])
@pytest.mark.parametrize("kind", ["held", "sched"])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("handle", ["10", "10_general", "20"])
def test_tick_bit_identical_to_staged_chain(a1, engines, handle, variant, kind, source):
    eng = engines[handle]
    N = eng.cfg.horizon
    B, T = 1024, 30
    got, want = _compare(a1, eng, _params(a1, VARIANTS[variant], kind, N), B, T, 61 + VARIANTS[variant], [source] * T)
    assert first_difference(got, want) is None, first_difference(got, want)
    modes = np.array([g["movement_mode"] for g in got])
    assert modes[:5].sum() == 0 and modes[5:].sum() > 0 and (modes[-1] == 0).any()     # standstill, walking, toggled out
    print("%s %s N=%d %s: %d ticks bit-identical, status per tick %s" % (handle, kind, N, variant, T, _status_counts(got)[-3:]))


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_large_batch_bit_identical(a1, engines, kind):
    eng = engines["10"]
    B, T = 65536, 3
    got, want = _compare(a1, eng, _params(a1, a1.VARIANT_GAZEBO, kind, 10), B, T, 11, [ESTIMATED] * T)
    assert first_difference(got, want) is None, first_difference(got, want)
    print("B=%d %s estimated: status counts per tick %s" % (B, kind, _status_counts(got)))


# ---- 3. against the oracle -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def loop43():
    return tick_solve_inputs(512, 64, 43, 10)


def _terrain_frame(n):
    """[B,4,3,3] the oracle's terrain_frame of unit normals n [B,4,3]: the rotation taking world z to n"""
    nx, ny, nz = n[..., 0], n[..., 1], n[..., 2]
    k = 1.0 / (1.0 + nz)
    R = np.zeros(n.shape[:-1] + (3, 3))
    R[..., 0, 0], R[..., 0, 1], R[..., 0, 2] = 1 - nx * nx * k, -nx * ny * k, nx
    R[..., 1, 0], R[..., 1, 1], R[..., 1, 2] = -nx * ny * k, 1 - ny * ny * k, ny
    R[..., 2, 0], R[..., 2, 1], R[..., 2, 2] = -nx, -ny, nz
    return R


def pyramid_excess(f_body, rot, normals, mask, mu, fz_max):
    """[B] largest violation (N) of any stance foot's terrain pyramid by the world force f, f_body = R^T f: |f'_x|, |f'_y| <= mu f'_z,
    0 <= f'_z <= fz_max in the foot's terrain frame (f' = Rf^T f, the oracle's terrain_frame).  R is solved against, not transposed: the
    orientation stage does not normalise the quaternion, so rot is orthogonal only to rounding of its norm"""
    B = f_body.shape[1]
    Rt = rot.T.reshape(B, 3, 3).transpose(0, 2, 1)
    f = np.linalg.solve(Rt, f_body.T.reshape(B, 4, 3).transpose(0, 2, 1)).transpose(0, 2, 1)
    n = normals.T.reshape(B, 4, 3)
    fl = np.einsum("blji,blj->bli", _terrain_frame(n / np.linalg.norm(n, axis=2, keepdims=True)), f)
    ex = np.maximum.reduce([np.abs(fl[..., 0]) - mu * fl[..., 2], np.abs(fl[..., 1]) - mu * fl[..., 2], -fl[..., 2], fl[..., 2] - fz_max])
    stance = ((mask[:, None] >> np.arange(4)[None, :]) & 1).astype(bool)
    return np.where(stance, ex, -np.inf).max(axis=1)


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_against_oracle(a1, O, loop43, kind):
    D = loop43
    B, T, N = 512, 64, 10
    tp = _params(a1, a1.VARIANT_GAZEBO, kind, N)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    tp.rho_opt[:], tp.rho_fix[:] = D["rho_opt"].tolist(), D["rho_fix"].tolist()
    tp.kp_foot[:], tp.kd_foot[:], tp.km_foot[:], tp.torques_gravity[:] = KP_ROS.tolist(), KD_ROS.tolist(), km.tolist(), tg.tolist()
    tp.use_terrain_adapt, tp.assume_flat_ground = 1, 1
    eng = _engine(a1, N)
    ds = DeviceSeqs(a1, eng, D["seqs"], D["speed"])
    try:
        chain = staged_chain_terrain(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T, record=True)
        got = tick_run_terrain(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T)
        assert first_difference(got, [{k: c[k] for k in OUT_SPECS} for c in chain]) is None
        cat = lambda k: np.ascontiguousarray(np.concatenate([c[k] for c in chain], axis=-1))
        st = dict(x0=cat("x0"), rot=cat("rot"), foot=cat("foot"), ref=cat("ref"), contact=cat("contacts"))
        sched, normals, f, status = cat("sched"), cat("normals"), cat("f_body"), cat("status")
        # the world-z solve of the same QPs, for the census
        fz, sz, _ = eng.solve_ext(st, sched, None)
    finally:
        ds.free()
        eng.close()
    # the device chain is the closed loop of the oracle chain
    for t in range(T):
        assert np.array_equal(chain[t]["contacts"], D["contact"][t]) and np.array_equal(chain[t]["movement_mode"], D["mode"][t]), t
        assert np.abs(chain[t]["x0"] - D["x0"][t]).max() <= 1e-8, t
    fo, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (info[:, 1] == 1).all()
    ef = np.abs(f - fo).max(axis=0)
    bad = np.nonzero((status != a1.STATUS_OPTIMAL) | ~(ef <= TOL_ORACLE))[0]
    assert bad.size == 0, "%d QPs fail (status %s, |f - f*| %s)" % (bad.size, status[bad][:8].tolist(), ef[bad][:8].tolist())
    cfg = a1.default_config()
    ex = pyramid_excess(f, st["rot"], normals, sched[0], cfg.mu, cfg.fz_max)
    assert ex.max() <= TOL_PYRAMID, ex.max()
    assert (sz == a1.STATUS_OPTIMAL).all()
    exz = pyramid_excess(fz, st["rot"], normals, sched[0], cfg.mu, cfg.fz_max)
    tilt = np.arccos(np.clip(normals[2], -1.0, 1.0))
    print("%s tick, estimated terrain, N=%d, %d QPs: every QP OPTIMAL, |f - f_oracle| max %.2e N, pyramid excess max %.2e N; normal tilt "
          "median %.3f max %.3f rad; world-z solutions outside the terrain pyramid: %d robot-ticks (%d by more than 1 N), worst %.2f N" % (
              kind, N, B * T, float(ef.max()), float(ex.max()), float(np.median(tilt)), float(tilt.max()), int((exz > TOL_PYRAMID).sum()),
              int((exz > 1.0).sum()), float(exz.max())))


# ---- 4. FLAT ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["held", "sched"])
def test_flat_is_the_tick_without_terrain(a1, engines, kind):
    eng = engines["10"]
    B, T = 1024, 30
    tp = _params(a1, a1.VARIANT_GAZEBO, kind, 10)
    seqs, speed = tick_inputs(B, T, 21)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    runs = {}
    try:
        for how in ("never", "flat", "estimated_then_flat", "estimated"):
            tick = a1.Tick(eng, B, tp)
            try:
                if how == "flat":
                    tick.set_terrain(a1.TERRAIN_FLAT)
                elif how == "estimated_then_flat":
                    tick.set_terrain(a1.TERRAIN_ESTIMATED)
                    tick.set_terrain(a1.TERRAIN_FLAT)
                elif how == "estimated":
                    tick.set_terrain(a1.TERRAIN_ESTIMATED)
                runs[how] = tick_run_device(a1, eng, tick, ds, B, T, DT)
            finally:
                tick.close()
        chain = staged_chain_terrain(a1, eng, tp, ds, B, T, DT, [ESTIMATED] * T, record=True)   # the run's estimated normals
    finally:
        ds.free()
    for how in ("flat", "estimated_then_flat"):
        assert first_difference(runs[how], runs["never"]) is None, (how, first_difference(runs[how], runs["never"]))
    assert first_difference([{k: c[k] for k in OUT_SPECS} for c in chain], runs["estimated"]) is None
    # the state does not depend on the forces: every tick of the two runs poses the same QPs, and where the normal is exactly e_z
    # (low body, the all-zero start) they are the same QP solved by another kernel
    worst, n = 0.0, 0
    for t in range(T):
        ez = (chain[t]["normals"][0:3] == np.array([[0.0], [0.0], [1.0]])).all(axis=0)
        g, w = runs["estimated"][t], runs["never"][t]
        assert np.array_equal(g["x0"], w["x0"]) and np.array_equal(g["ref"], w["ref"]) and np.array_equal(g["contacts"], w["contacts"]), t
        assert (g["status"][ez] == a1.STATUS_OPTIMAL).all() and (w["status"][ez] == a1.STATUS_OPTIMAL).all(), t
        if ez.any():
            worst = max(worst, float(np.abs(g["f_body"][:, ez] - w["f_body"][:, ez]).max()))
            n += int(ez.sum())
    print("%s: FLAT bit-identical to the tick without terrain; %d robot-ticks with n = e_z, |f_estimated - f_flat| max %.2e N" % (kind, n, worst))
    assert n >= B and worst <= 1e-8


# ---- 5. reset and switching ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["held", "sched"])
def test_reset_robots_gives_fresh_terrain_ticks(a1, engines, kind):
    eng = engines["10"]
    B, T, tr = 1024, 30, 14
    tp = _params(a1, a1.VARIANT_GAZEBO, kind, 10)
    seqs, speed = tick_inputs(B, T, 31)
    mask = np.random.default_rng(32).random(B) < 0.25
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        src = [ESTIMATED] * T
        a = tick_run_terrain(a1, eng, tp, ds, B, T, DT, src, resets={tr: mask})
        u = tick_run_terrain(a1, eng, tp, ds, B, T, DT, src)
        f = tick_run_terrain(a1, eng, tp, ds, B, T, DT, src, t0=tr)
        # a1mpc_tick_reset keeps the source and reproduces the first ticks
        tick = a1.Tick(eng, B, tp)
        try:
            tick.set_terrain(a1.TERRAIN_ESTIMATED)
            first = tick_run_device(a1, eng, tick, ds, B, 12, DT)
            tick.reset()
            again = tick_run_device(a1, eng, tick, ds, B, 12, DT)
        finally:
            tick.close()
    finally:
        ds.free()
    assert first_difference(a[:tr], u[:tr]) is None
    for t in range(tr, T):
        for k in OUT_SPECS:
            assert a[t][k][..., mask].tobytes() == f[t - tr][k][..., mask].tobytes(), (t, k, "reset robots")
            assert a[t][k][..., ~mask].tobytes() == u[t][k][..., ~mask].tobytes(), (t, k, "other robots")
    assert first_difference(again, first) is None
    assert first_difference(first, u[:12]) is None


@pytest.mark.parametrize("kind", ["held", "sched"])
def test_switching_source_mid_run(a1, engines, kind):
    eng = engines["10"]
    B, T = 1024, 30
    sources = [FLAT] * 8 + [ESTIMATED] * 8 + [GIVEN] * 4 + [FLAT] * 4 + [ESTIMATED] * 6
    got, want = _compare(a1, eng, _params(a1, a1.VARIANT_ISAAC, kind, 10), B, T, 41, sources)
    assert first_difference(got, want) is None, first_difference(got, want)


# ---- 6. argument errors ----------------------------------------------------------------------------------------------------------

def test_argument_errors(a1, engines):
    L = a1.lib()
    eng = engines["10"]
    B = 64
    buf = np.zeros((12, B))
    d_nrm = eng.dalloc(12 * B * 8)
    qp = a1.Tick(eng, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP))
    mpc = a1.Tick(eng, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC))
    e_aniso = _engine(a1, 10, r=[1e-7, 2e-7, 1e-7] * 4)
    aniso = a1.Tick(e_aniso, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC))
    sw = eng.swing_alloc(B)
    try:
        err = lambda: L.a1mpc_last_error()
        assert L.a1mpc_tick_set_terrain(qp.t, ESTIMATED, None) == -1 and b"MPC mode" in err()
        assert L.a1mpc_tick_set_terrain(qp.t, GIVEN, d_nrm) == -1
        assert L.a1mpc_tick_set_terrain(qp.t, FLAT, None) == 0
        for s in (-1, 3, 100):
            assert L.a1mpc_tick_set_terrain(mpc.t, s, None) == -1 and b"unknown terrain source" in err()
        assert L.a1mpc_tick_set_terrain(mpc.t, GIVEN, None) == -1 and b"needs a normals array" in err()
        assert L.a1mpc_tick_set_terrain(mpc.t, GIVEN, buf.ctypes.data) == -1 and b"device memory" in err()
        assert L.a1mpc_tick_set_terrain(aniso.t, ESTIMATED, None) == -1 and b"isotropic" in err()
        assert L.a1mpc_tick_set_terrain(aniso.t, GIVEN, d_nrm) == -1 and b"isotropic" in err()
        assert L.a1mpc_tick_set_terrain(aniso.t, FLAT, None) == 0
        assert L.a1mpc_tick_set_terrain(mpc.t, GIVEN, d_nrm) == 0 and L.a1mpc_tick_set_terrain(mpc.t, ESTIMATED, d_nrm) == 0
        # a1mpc_terrain_normals_batch
        pos, ref, pitch = np.full((3, B), 0.3), np.zeros((9, B)), np.zeros(B)
        P = lambda a: a.ctypes.data
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 1, P(pos), P(ref), B, P(pitch), None) == -1              # normals required
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 1, P(pos), None, B, None, P(buf)) == -1                  # adaptation needs ref
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 0, None, None, B, None, P(buf)) == -1                    # root_pos required
        assert L.a1mpc_terrain_normals_batch(eng.h, 0, sw, 0, P(pos), None, B, None, P(buf)) == -1
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 1, P(pos), P(ref), B - 1, None, P(buf)) == -1            # ld < B
        assert L.a1mpc_terrain_normals_batch(eng.h, B, P(buf), 0, P(pos), None, B, None, P(buf)) == -1              # host state
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 0, P(pos), None, B, None, d_nrm) == -1                   # mixed sides
        assert L.a1mpc_terrain_normals_batch(eng.h, B, sw, 0, P(pos), None, B, None, P(buf)) == 0
        assert (buf[2::3] == 1.0).all()                                                                             # fresh state: flat
        # after the rejected calls the ticks still run
        seqs, speed = tick_inputs(B, 2, 9)
        for tk in (mpc, qp, aniso):
            tau, o = tk.run(DT, *(seqs[n][0] for n in a1.TICK_INPUTS[:-1]), speed)
            assert np.isfinite(tau).all() and (o["status"] == a1.STATUS_OPTIMAL).all()
    finally:
        for tk in (qp, mpc, aniso):
            tk.close()
        e_aniso.close()
        L.a1mpc_device_free(eng.h, d_nrm)
        L.a1mpc_device_free(eng.h, sw)
