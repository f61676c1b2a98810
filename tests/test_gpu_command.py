"""-m gpu: a1mpc_orientation_batch and a1mpc_command_batch (the adapters' orientation stage and main_update's front half) on the H100:
the fixture (tests/golden/command_v1.npz) through host and device pointers; outputs written straight into x0 / ref rows with ld > B,
every row the calls do not own left bit-identical; and a whole control tick from raw sensor arrays on device pointers, in MPC and QP
mode, against the same chain of oracle stages.

Tolerances: tests/command_scenarios.py for the two stages (rot <= 4e-16, euler <= 1e-15 rad with yaw modulo 2 pi, rot_z <= 4e-16 +
|yaw error|, filters and root_ang_vel <= 1e-15 relative, movement_mode exact).  In the closed loop: contacts and movement_mode exact;
the estimator's x0 rows <= 1e-8; forces <= 1e-4 N with every QP OPTIMAL; torques as the other closed-loop tests."""
import ctypes as C
import os

import numpy as np
import pytest

from command_scenarios import (DT, HEIGHT0, HMAX, HMIN, KP_LINEAR, KP_LOCK, VARIANTS, check_command, check_orientation, command_sequence,
                               imu_sequence)
from common import estimation_scenario
from oracle import command_oracle_py as CO
from oracle import swing_oracle_py as SO
from stance_scenarios import gains, oracle_forces, root_acc_batch
from swing_scenarios import CPS, KD_ROS, KP_ROS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 10


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
    e = a1.Engine(a1.default_config(horizon=N))
    yield e
    e.close()


@pytest.fixture(scope="module")
def G():
    with np.load(os.path.join(ROOT, "tests", "golden", "command_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _h2d(a1, eng, ptr, x):
    x = np.ascontiguousarray(x)
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, ptr, x.ctypes.data, x.nbytes))


def _d2h(a1, eng, ptr, shape, dtype=np.float64):
    x = np.zeros(shape, dtype=dtype)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, x.ctypes.data, ptr, x.nbytes))
    eng.sync()
    return x


def _off(ptr, nbytes):
    return C.c_void_p(ptr.value + nbytes)


def _params(a1, v):
    cp = a1.default_command_params(v)
    assert (cp.body_height, cp.body_height_min, cp.body_height_max) == (HEIGHT0[v], HMIN, HMAX)
    assert tuple(cp.kp_linear) == KP_LINEAR and tuple(cp.kp_linear_lock) == KP_LOCK
    return cp


def _records(G, v, t):
    o = {k: G[k][v, t] for k in ("rot", "rot_z", "euler", "ang_vel", "imu_acc", "imu_ang_vel")}
    c = tuple(G[k][v, t] for k in ("movement_mode", "kp_linear", "ref", "des"))
    return o, c


def test_fixture_host_pointers(a1, eng, G):
    _, T, _, R = G["quat"].shape
    for v in VARIANTS:
        imu = eng.imu_alloc(R) if v != 1 else None
        ref = np.full((9, R), np.nan)
        cs = eng.command_alloc(R, _params(a1, v), ref)
        assert (ref == 0.0).all()
        for t in range(T):
            o = eng.orientation(G["quat"][v, t], G["gyro"][v, t], G["acc"][v, t], imu)
            o0, c0 = _records(G, v, t)
            check_orientation(o, o0, "host variant %d tick %d" % (v, t))
            ov = G["pitch_override"][v, t]
            ref[1] = np.where(np.isnan(ov), ref[1], ov)
            mode, kp, des = eng.command(cs, DT, G["cmd"][v, t], G["root_pos"][v, t], ref)
            check_command((mode, kp, ref, des), c0, "host variant %d tick %d" % (v, t))
        for p in (imu, cs):
            if p is not None:
                a1.lib().a1mpc_device_free(eng.h, p)


def test_fixture_device_pointers(a1, eng, G):
    L = a1.lib()
    _, T, _, R = G["quat"].shape
    names = dict(quat=4, gyro=3, acc=3, cmd=7, root_pos=3)
    for v in VARIANTS:
        # the whole sequence on the device before the first tick; per tick the calls index into it
        din = {k: eng.dalloc(T * n * R * 8) for k, n in names.items()}
        for k in names:
            _h2d(a1, eng, din[k], G[k][v])
        ov = G["pitch_override"][v]
        d = {k: eng.dalloc(n * R * 8) for k, n in dict(rot=9, rz=9, x0=12, ia=3, ig=3, kp=3, ref=9, des=12).items()}
        d_mode = eng.dalloc(R * 4)
        imu = eng.imu_alloc(R) if v != 1 else None
        cs = eng.dalloc(L.a1mpc_command_bytes(R))
        a1._check(L.a1mpc_command_init_batch(eng.h, R, cs, C.byref(_params(a1, v)), d["ref"], R))
        for t in range(T):
            a1._check(L.a1mpc_orientation_batch(eng.h, R, _off(din["quat"], t * 4 * R * 8), _off(din["gyro"], t * 3 * R * 8),
                                                _off(din["acc"], t * 3 * R * 8), imu, d["rot"], d["rz"], d["x0"], R, d["ia"], d["ig"]))
            if not np.isnan(ov[t]).all():   # what the terrain stage leaves in row 1
                row = _d2h(a1, eng, _off(d["ref"], R * 8), R)
                _h2d(a1, eng, _off(d["ref"], R * 8), np.where(np.isnan(ov[t]), row, ov[t]))
            a1._check(L.a1mpc_command_batch(eng.h, R, cs, DT, _off(din["cmd"], t * 7 * R * 8), _off(din["root_pos"], t * 3 * R * 8), R, d_mode,
                                            d["kp"], d["ref"], R, d["des"], R))
            x0 = _d2h(a1, eng, d["x0"], (12, R))
            o = dict(rot=_d2h(a1, eng, d["rot"], (9, R)), rot_z=_d2h(a1, eng, d["rz"], (9, R)), euler=x0[0:3], ang_vel=x0[6:9],
                     imu_acc=_d2h(a1, eng, d["ia"], (3, R)), imu_ang_vel=_d2h(a1, eng, d["ig"], (3, R)))
            o0, c0 = _records(G, v, t)
            check_orientation(o, o0, "device variant %d tick %d" % (v, t))
            c = (_d2h(a1, eng, d_mode, R, np.uint32), _d2h(a1, eng, d["kp"], (3, R)), _d2h(a1, eng, d["ref"], (9, R)), _d2h(a1, eng, d["des"], (12, R)))
            check_command(c, c0, "device variant %d tick %d" % (v, t))
        for p in list(din.values()) + list(d.values()) + [d_mode, cs] + ([imu] if imu is not None else []):
            L.a1mpc_device_free(eng.h, p)


def test_rows_written_in_place_with_ld(a1, eng, G):
    """ld > B: outputs straight into x0 rows 0-2 / 6-8, rot, rot_z, ref and the stance arrays; everything else keeps its sentinel"""
    L = a1.lib()
    v, t = 0, 40
    R = G["quat"].shape[3]
    B, ld = R, R + 5
    S = 7.25
    for device in (False, True):
        x0 = np.full((12, ld), S); rot = np.full((9, ld), S); rz = np.full((9, ld), S); ref = np.full((9, ld), S)
        des = np.full((12, ld), S); kp = np.full((3, ld), S)
        x0[3:6, :B] = G["root_pos"][v, t]
        quat, gyro, acc, cmd = (np.ascontiguousarray(G[k][v, t]) for k in ("quat", "gyro", "acc", "cmd"))
        mode = np.zeros(B, dtype=np.uint32)
        cs = eng.dalloc(L.a1mpc_command_bytes(B))
        a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(_params(a1, v)), None, B))
        ref[1, :B] = 0.0
        arrays = dict(x0=x0, rot=rot, rz=rz, ref=ref, des=des, kp=kp, quat=quat, gyro=gyro, acc=acc, cmd=cmd, mode=mode)
        if device:
            dp = {k: eng.dalloc(a.nbytes) for k, a in arrays.items()}
            for k, a in arrays.items():
                _h2d(a1, eng, dp[k], a)
            P = lambda k: dp[k]
        else:
            P = lambda k: C.c_void_p(arrays[k].ctypes.data)
        a1._check(L.a1mpc_orientation_batch(eng.h, B, P("quat"), P("gyro"), P("acc"), None, P("rot"), P("rz"), P("x0"), ld, None, None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, DT, P("cmd"), _off(P("x0"), 3 * ld * 8), ld, P("mode"),
                                        P("kp"), P("ref"), ld, P("des"), ld))
        if device:
            for k, a in arrays.items():
                arrays[k] = _d2h(a1, eng, dp[k], a.shape, a.dtype)
            for p in dp.values():
                L.a1mpc_device_free(eng.h, p)
        eng.sync()
        L.a1mpc_device_free(eng.h, cs)
        x0, rot, rz, ref, des, kp, mode = (arrays[k] for k in ("x0", "rot", "rz", "ref", "des", "kp", "mode"))
        what = "device" if device else "host"
        for a in (x0, rot, rz, ref, des, kp):
            assert (a[:, B:] == S).all(), what                                  # the columns past B
        assert (x0[9:12] == S).all() and np.array_equal(x0[3:6, :B], G["root_pos"][v, t]), what   # the estimator's rows
        o = CO.Orientation(B, filtered=False)(quat, gyro)
        check_orientation(dict(rot=rot[:, :B], rot_z=rz[:, :B], euler=x0[0:3, :B], ang_vel=x0[6:9, :B], imu_acc=None, imu_ang_vel=o["imu_ang_vel"]),
                          o, what)
        c0 = CO.Command(B, v, HEIGHT0[v], HMIN, HMAX, KP_LINEAR, KP_LOCK)(DT, cmd, G["root_pos"][v, t], np.zeros(B))
        check_command((mode, kp[:, :B], ref[:, :B], des[:, :B]), c0, what)


def test_argument_errors(a1, eng):
    L = a1.lib()
    B = 8
    z = lambda *s: np.zeros(s)
    P = lambda a: a.ctypes.data
    q, g, a, cmd, pos = z(4, B), z(3, B), z(3, B), z(7, B), z(3, B)
    rot, x0, mode, kp, ref = z(9, B), z(12, B), np.zeros(B, dtype=np.uint32), z(3, B), z(9, B)
    imu, cs = eng.imu_alloc(B), eng.command_alloc(B)
    host_state = z(64 * B)
    ori = lambda **k: L.a1mpc_orientation_batch(eng.h, k.get("B", B), k.get("q", P(q)), P(g), k.get("a", P(a)), k.get("imu", imu), P(rot), None,
                                                k.get("x0", P(x0)), k.get("ld", B), k.get("ia", None), None)
    com = lambda **k: L.a1mpc_command_batch(eng.h, k.get("B", B), k.get("cs", cs), k.get("dt", DT), P(cmd), k.get("pos", P(pos)), k.get("pld", B),
                                            P(mode), k.get("kp", P(kp)), P(ref), k.get("rld", B), None, k.get("sld", B))
    assert ori() == 0 and com() == 0
    assert ori(imu=None) == 0
    assert ori(imu=P(host_state)) == -1 and b"device memory" in L.a1mpc_last_error()
    assert com(cs=P(host_state)) == -1 and b"device memory" in L.a1mpc_last_error()
    assert ori(a=None, ia=P(a)) == -1                                 # imu_acc needs acc
    for nb in (0, -1):
        assert ori(B=nb) == -1 and com(B=nb) == -1
        assert L.a1mpc_imu_init_batch(eng.h, nb, imu) == -1
        assert L.a1mpc_command_init_batch(eng.h, nb, cs, C.byref(a1.default_command_params()), None, B) == -1
    assert ori(ld=B - 1) == -1 and com(pld=B - 1) == -1 and com(rld=B - 1) == -1 and com(sld=B - 1) == -1
    assert ori(q=None) == -1 and com(pos=None) == -1 and com(kp=None) == -1 and com(dt=0.0) == -1
    d = eng.dalloc(4 * B * 8)
    assert ori(q=d) == -1 and b"all-host or all-device" in L.a1mpc_last_error()
    assert com(pos=d) == -1 and b"all-host or all-device" in L.a1mpc_last_error()
    bad = a1.default_command_params(); bad.variant = 3
    assert L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(bad), None, B) == -1 and b"variant" in L.a1mpc_last_error()
    assert L.a1mpc_command_init_batch(eng.h, B, P(host_state), C.byref(a1.default_command_params()), None, B) == -1
    assert L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(a1.default_command_params()), P(ref), B - 1) == -1
    assert L.a1mpc_imu_init_batch(eng.h, B, P(host_state)) == -1
    for p in (imu, cs, d):
        L.a1mpc_device_free(eng.h, p)


def _closed_loop(a1, O, eng, qp_mode, B=1024, T=30, seed=41):
    """every stage of a tick on device pointers, no host copy inside a tick: orientation -> leg kinematics -> command -> update_plan ->
    swing legs -> EKF (into x0 rows 3-5 / 9-11, ld = B) -> terrain pitch (MPC) -> solve or stance QP -> joint torques.  The MPC solve is
    a1mpc_solve_batch_ext_warm without a schedule: the contact pattern held over the horizon, as compute_grf poses it."""
    L = a1.lib()
    rng = np.random.default_rng(seed)
    mass, kdl, kpa, kda = gains("gazebo")
    _, rho_opt, rho_fix, _, _, _ = estimation_scenario(4, 5)
    rho_opt, rho_fix = np.ascontiguousarray(rho_opt.reshape(12)), np.ascontiguousarray(rho_fix.reshape(20))
    quat, gyro, acc = imu_sequence(B, T, seed, gimbal_share=0.0, gentle=True)
    cmd, _ = command_sequence(B, T, seed + 1)
    cmd[:, 6] = 0.0
    cmd[5, 6] = 1.0                                                 # standstill, then walking from tick 5; later toggles out and back
    cmd[18, 6, : B // 2] = 1.0
    cmd[24, 6, : B // 4] = 1.0
    cmd[:, 4] = np.where(np.arange(B) % 2 == 0, 0.3, -0.2)[None, :]   # a non-zero pitch rate on top of the terrain pitch
    q = np.tile(np.array([0.0, 0.8, -1.6] * 4)[None, :, None], (T, 1, B)) + 0.05 * rng.standard_normal((T, 12, B))
    dq = 0.5 * rng.standard_normal((T, 12, B))
    force = rng.uniform(0.0, 80.0, (T, 4, B))
    speed = np.repeat(rng.choice([2.0, 3.0, 4.0], B)[None, :], 4, axis=0)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    kp, kd = KP_ROS.copy(), KD_ROS.copy()
    gp = a1.default_gait_params(N)
    cp = a1.default_command_params(a1.VARIANT_GAZEBO)
    # device buffers: the whole run's raw sensor and command arrays are uploaded before the first tick
    seqs = dict(quat=quat, gyro=gyro, acc=acc, cmd=cmd, q=q, dq=dq, force=force)
    ds = {k: eng.dalloc(v.nbytes) for k, v in seqs.items()}
    for k, v in seqs.items():
        _h2d(a1, eng, ds[k], v)
    at = lambda k, t: _off(ds[k], t * seqs[k][0].nbytes)
    d = a1.DeviceBatch(eng, B)
    _h2d(a1, eng, d.x0, np.zeros((12, B)))
    nb = dict(rz=9, ia=3, ig=3, fpr=12, fvr=12, jac=36, kpl=3, des=12, gc=4, sp=4, trel=12, fk=12, tau=12, pos=3, vel=3)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    _h2d(a1, eng, dv["gc"], np.zeros((4, B))); _h2d(a1, eng, dv["sp"], speed); _h2d(a1, eng, dv["tau"], np.zeros((12, B)))
    d_mode, d_plan, d_sched, d_est, d_est_status = eng.dalloc(B * 4), eng.dalloc(B * 4), eng.dalloc(N * B * 4), eng.dalloc(B * 4), eng.dalloc(B * 4)
    imu, sw, ekf, warm = eng.imu_alloc(B), eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B)), eng.warm_alloc(B)
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(cp), d.ref, B))
    x0p = lambda row: _off(d.x0, row * B * 8)
    # the CPU chain
    ori, com, ora = CO.Orientation(B), CO.Command(B, 0, cp.body_height, HMIN, HMAX, KP_LINEAR, KP_LOCK), SO.Swing(B)
    ocfg = O.make_config(horizon=N)
    x0o = np.zeros((12, B)); gc0 = np.zeros((4, B)); tau0 = np.zeros((12, B))
    xs = [None] * B; Ps = [None] * B
    row1 = np.zeros(B)
    worst = dict(f=0.0, tau=0.0, x0=0.0)
    seen = dict(walk=0, leave=0, yaw_wrap=False, adapt=False)
    yaw_prev = None
    for t in range(T):
        # ---- one tick on the device ----
        a1._check(L.a1mpc_orientation_batch(eng.h, B, at("quat", t), at("gyro", t), at("acc", t), imu, d.rot, dv["rz"], d.x0, B, dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, at("q", t), at("dq", t), d.rot, rho_opt.ctypes.data, rho_fix.ctypes.data, dv["fpr"],
                                               dv["jac"], dv["fvr"], d.foot, None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, DT, at("cmd", t), x0p(3), B, d_mode, dv["kpl"], None if qp_mode else d.ref, B, dv["des"], B))
        lvd = _off(dv["des"], 6 * B * 8) if qp_mode else _off(d.ref, 5 * B * 8)
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(gp), dv["gc"], dv["sp"], d_mode, x0p(9), lvd, dv["rz"], d.rot, x0p(3), d_plan, d_sched,
                                            dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, DT, dv["gc"], d_plan, dv["rz"], d.foot,
                                           dv["trel"], at("force", t), dv["fk"], d.contact, None, None))
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], d.rot))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, DT, 1, d_mode, dv["ia"], dv["ig"], d.rot, dv["fpr"], dv["fvr"], at("force", t), x0p(3),
                                               x0p(9), d_est, d_est_status))
        if qp_mode:
            a1._check(L.a1mpc_stance_qp_batch(eng.h, B, C.c_size_t(B), d.x0, d.rot, dv["rz"], d.foot, d.contact, dv["des"], dv["kpl"], kdl.ctypes.data,
                                              kpa.ctypes.data, kda.ctypes.data, d.f_body, d.status, None))
        else:
            a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, x0p(3), d.ref, B, None))
            a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), None, C.byref(d.out), warm, 0))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, d.f_body, dv["fk"], dv["jac"], d.contact, km.ctypes.data, tg.ctypes.data, dv["tau"]))
        f, status = d.download()
        x0 = _d2h(a1, eng, d.x0, (12, B))
        con, mode, tau = _d2h(a1, eng, d.contact, B, np.uint32), _d2h(a1, eng, d_mode, B, np.uint32), _d2h(a1, eng, dv["tau"], (12, B))
        # ---- the same tick from oracle stages ----
        o = ori(quat[t], gyro[t], acc[t])
        x0o[0:3], x0o[6:9] = o["euler"], o["ang_vel"]
        R = o["rot"].T.reshape(B, 3, 3)
        p = np.zeros((B, 4, 3)); J = np.zeros((B, 4, 3, 3))
        for b in range(B):
            for leg in range(4):
                p[b, leg], J[b, leg] = O.leg_kinematics(q[t, 3 * leg:3 * leg + 3, b], rho_opt[3 * leg:3 * leg + 3], rho_fix[5 * leg:5 * leg + 5])
        fpr = p.reshape(B, 12).T.copy()
        fvr = np.stack([np.einsum("bij,jb->ib", J[:, leg], dq[t, 3 * leg:3 * leg + 3]) for leg in range(4)]).reshape(12, B)
        fabs = np.einsum("bij,blj->bli", R, p).reshape(B, 12).T.copy()
        mode0, kpl0, ref0, des0 = com(DT, cmd[t], x0o[3:6], None if qp_mode else row1)
        plan0 = np.zeros(B, dtype=np.uint32); sched0 = np.zeros((N, B), dtype=np.uint32); trel0 = np.zeros((12, B))
        for b in range(B):
            gc0[:, b], plan0[b], sched0[:, b], trel0[:, b], _, _ = O.update_plan(gp, mode0[b], gc0[:, b], speed[:, b], x0o[9:12, b], ref0[5:8, b],
                                                                                 o["rot_z"][:, b], o["rot"][:, b], x0o[3:6, b])
        fk0, con0, _, _ = ora.legs(CPS, DT, kp, kd, gc0, plan0, o["rot_z"], fabs, trel0, force[t])
        for b in range(B):
            if t == 0:
                xs[b], Ps[b] = O.ekf_init(fpr[:, b], o["rot"][:, b])
            else:
                xs[b], Ps[b], x0o[3:6, b], x0o[9:12, b], _, rc = O.ekf_update(xs[b], Ps[b], DT, 1, mode0[b], o["imu_acc"][:, b], o["imu_ang_vel"][:, b],
                                                                              o["rot"][:, b], fpr[:, b], fvr[:, b], force[t, :, b])
                assert rc == 0
        if qp_mode:
            acc0 = root_acc_batch(x0o, o["rot"], des0, kpl0, kdl, kpa, kda, mass)
            fo, ok = oracle_forces(O, acc0, o["rot_z"], o["rot"], fabs, con0)
            assert ok.all()
        else:
            ora.terrain(1, x0o[3:6], ref0)
            row1 = ref0[1].copy()
            fo, info = O.compute_grf_batch_ext(ocfg, O.Batch(x0o, o["rot"], fabs, ref0, con0), None, None, O.MODE_EXACT, nthreads=O.hardware_threads())
        for b in range(B):
            tau0[:, b] = O.joint_torques(fo[:, b], fk0[:, b], J[b].reshape(36), int(con0[b]), km, tg, tau0[:, b])
        # ---- compare ----
        assert np.array_equal(mode, mode0) and np.array_equal(con, con0), t
        ex = float(np.abs(x0 - x0o).max())
        assert ex <= 1e-8, (t, ex)
        if qp_mode:
            stance = (con & 15) != 0
            assert (status[stance] == a1.STATUS_OPTIMAL).all() and (status[~stance] == a1.STATUS_NO_CONTACT).all(), (t, np.bincount(status))
        else:
            bad = np.nonzero(status != a1.STATUS_OPTIMAL)[0]
            assert bad.size == 0, (t, np.bincount(status), bad, x0[:, bad].T, _d2h(a1, eng, d.ref, (9, B))[:, bad].T, con[bad], sched0[:, bad].T)
        ef = float(np.abs(f - fo).max())
        assert ef <= 1e-4, (t, ef)
        jn = np.abs(J).sum(axis=2).reshape(B, 12).T
        et = float((np.abs(tau - tau0) - (1e-4 * jn + 1e-8 * np.maximum(1.0, np.abs(tau0)))).max())
        assert et <= 0.0, (t, et)
        worst = dict(f=max(worst["f"], ef), tau=max(worst["tau"], float(np.abs(tau - tau0).max())), x0=max(worst["x0"], ex))
        seen["walk"] += int(mode.sum())
        if t > 0:
            seen["leave"] += int(((mode0 == 0) & (prev_mode == 1)).sum())
            seen["yaw_wrap"] |= bool((np.abs(x0o[2] - yaw_prev) > np.pi).any())
        if not qp_mode:
            seen["adapt"] |= bool((ref0[1] != 0.0).any())
        prev_mode, yaw_prev = mode0.copy(), x0o[2].copy()
    assert seen["walk"] > 0 and seen["leave"] > 0 and seen["yaw_wrap"], seen
    d.free()
    for p in list(ds.values()) + list(dv.values()) + [d_mode, d_plan, d_sched, d_est, d_est_status, imu, sw, ekf, warm, cs]:
        L.a1mpc_device_free(eng.h, p)
    print("%s closed loop B=%d x %d ticks: |x0 - x0_oracle| %.2e, |f - f_oracle| %.2e N, |tau - tau_oracle| %.2e Nm, %s" % (
        "QP" if qp_mode else "MPC", B, T, worst["x0"], worst["f"], worst["tau"], seen))


def test_closed_loop_from_raw_arrays_mpc(a1, O, eng):
    _closed_loop(a1, O, eng, qp_mode=False)


def test_closed_loop_from_raw_arrays_qp(a1, O):
    mass = gains("gazebo")[0]
    e = a1.Engine(a1.default_config(horizon=N, mass=mass))
    try:
        _closed_loop(a1, O, e, qp_mode=True)
    finally:
        e.close()
