"""-m gpu: a1mpc_swing_legs_batch and a1mpc_terrain_pitch_batch (generate_swing_legs_ctrl and compute_grf's terrain adaptation) on the
H100: the reference's own vectors (tests/golden/swing_v1.npz), the oracle at B = 16 384 device-resident robots, a whole control tick
chained on device pointers (leg kinematics -> update_plan -> swing legs -> terrain pitch -> scheduled warm solve -> joint torques)
against the same chain of oracle stages, and argument errors.

Tolerances (tests/swing_scenarios.py): contacts exact; foot_pos_recent_contact bit-identical (additions in a fixed order and one IEEE
division); f_kin <= 1e-10 max(1, |f_kin|_inf) N; terrain_pitch and ref[1] <= 1e-7 rad -- acos near 1 (flat ground) turns rounding of the
cosine into ~1e-8 rad of angle."""
import ctypes as C
import os

import numpy as np
import pytest

from common import estimation_scenario
from oracle import swing_oracle_py as SO
from swing_scenarios import CPS, KD_RESET, KD_ROS, KP_RESET, KP_ROS, Scenario, check_tick

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = 0.0025
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


def _h2d(a1, eng, ptr, x):
    x = np.ascontiguousarray(x)
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, ptr, x.ctypes.data, x.nbytes))


def _d2h(a1, eng, ptr, shape, dtype):
    x = np.zeros(shape, dtype=dtype)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, x.ctypes.data, ptr, x.nbytes))
    eng.sync()
    return x


def _off(ptr, nbytes):
    return C.c_void_p(ptr.value + nbytes)


def test_golden_replay(a1, eng):
    """the reference's own records, every tick, through the host-pointer path"""
    with np.load(os.path.join(ROOT, "tests", "golden", "swing_v1.npz")) as z:
        G = {k: z[k] for k in z.files}
    gp = a1.default_gait_params(N)
    T = G["contacts"].shape[1]
    worst = [0.0, 0.0]
    for ids in ([0, 1, 2], [3, 4, 5]):
        B = len(ids)
        sw = eng.swing_alloc(B)
        for t in range(T):
            g = lambda k: np.ascontiguousarray(G[k][ids, t].T)
            fk, con, cur, rc = eng.swing_legs(gp, G["kp"][ids[0]], G["kd"][ids[0]], sw, DT, g("gait_counter"), G["plan_contacts"][ids, t], g("rot_z"),
                                              g("foot_pos_abs"), g("foot_pos_target_rel"), g("foot_force"))
            ref = np.zeros((9, B))
            pitch = eng.terrain_pitch(sw, 1, g("root_pos"), ref)
            ef, ea = check_tick((fk, con, rc, pitch, ref[1]), (g("f_kin"), G["contacts"][ids, t], g("foot_pos_recent_contact"), G["terrain_pitch"][ids, t],
                                                               G["root_euler_d1"][ids, t]), "robots %s tick %d" % (ids, t))
            worst = [max(worst[0], ef), max(worst[1], ea)]
        a1.lib().a1mpc_device_free(eng.h, sw)
    print("golden replay: f_kin rel %.2e, angle %.2e rad" % tuple(worst))


def test_oracle_parity_16384_device_resident(a1, O, eng):
    B, T = 16384, 300
    sc = Scenario(B, 91)
    ora = SO.Swing(B)
    sw = eng.swing_alloc(B)
    gp = a1.default_gait_params(N)
    L = a1.lib()
    sz = dict(gait_counter=4, rot_z=9, foot_pos_abs=12, foot_pos_target_rel=12, foot_force=4, root_pos=3)
    din = {k: eng.dalloc(n * B * 8) for k, n in sz.items()}
    d_plan, d_con = eng.dalloc(B * 4), eng.dalloc(B * 4)
    d_fk, d_rc, d_ref, d_pitch = eng.dalloc(12 * B * 8), eng.dalloc(12 * B * 8), eng.dalloc(9 * B * 8), eng.dalloc(B * 8)
    kp, kd = KP_RESET.copy(), KD_RESET.copy()
    worst = [0.0, 0.0]
    for t in range(T):
        x = sc.tick()
        for k in sz:
            _h2d(a1, eng, din[k], x[k])
        _h2d(a1, eng, d_plan, x["plan_contacts"])
        _h2d(a1, eng, d_ref, np.full((9, B), 3.0))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, DT, din["gait_counter"], d_plan, din["rot_z"],
                                           din["foot_pos_abs"], din["foot_pos_target_rel"], din["foot_force"], d_fk, d_con, None, d_rc))
        a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, din["root_pos"], d_ref, B, d_pitch))
        fk, con = _d2h(a1, eng, d_fk, (12, B), np.float64), _d2h(a1, eng, d_con, B, np.uint32)
        rc, ref, pitch = _d2h(a1, eng, d_rc, (12, B), np.float64), _d2h(a1, eng, d_ref, (9, B), np.float64), _d2h(a1, eng, d_pitch, B, np.float64)
        fk0, con0, _, rc0 = ora.legs(CPS, DT, kp, kd, x["gait_counter"], x["plan_contacts"], x["rot_z"], x["foot_pos_abs"], x["foot_pos_target_rel"],
                                     x["foot_force"])
        ref0 = np.full((9, B), 3.0)
        pitch0 = ora.terrain(1, x["root_pos"], ref0)
        ef, ea = check_tick((fk, con, rc, pitch, ref[1]), (fk0, con0, rc0, pitch0, ref0[1]), "tick %d" % t)
        assert np.array_equal(np.delete(ref, 1, axis=0), np.full((8, B), 3.0))
        worst = [max(worst[0], ef), max(worst[1], ea)]
    for p in list(din.values()) + [d_plan, d_con, d_fk, d_rc, d_ref, d_pitch, sw]:
        L.a1mpc_device_free(eng.h, p)
    print("oracle parity B=%d x %d ticks: f_kin rel %.2e, angle %.2e rad" % (B, T, *worst))


def _rz_rows(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    z, o = np.zeros_like(yaw), np.ones_like(yaw)
    return np.stack([c, -s, z, s, c, z, z, z, o])


def test_closed_loop_tick_on_device(a1, O, eng):
    """every stage of a control tick on device pointers, no host copy inside a tick; the same chain of oracle stages on the CPU"""
    B, T = 4096, 50
    L = a1.lib()
    rng = np.random.default_rng(23)
    _, rho_opt, rho_fix, _, _, _ = estimation_scenario(4, 5)
    rho_opt, rho_fix = np.ascontiguousarray(rho_opt.reshape(12)), np.ascontiguousarray(rho_fix.reshape(20))
    st = a1.gen_states(B, 2, 17)
    rot, x0, ref_in = st["rot"], st["x0"], st["ref"]
    rot_z = _rz_rows(x0[2])
    root_pos, lin_vel, lin_vel_d = x0[3:6].copy(), x0[9:12].copy(), ref_in[5:8].copy()
    speed = np.repeat(rng.choice([2.0, 3.0, 4.0], B)[None, :], 4, axis=0)
    mode = np.stack([np.full(B, 1 if t >= 5 else 0, dtype=np.uint32) for t in range(T)])
    q = np.tile(np.array([0.0, 0.8, -1.6] * 4)[None, :, None], (T, 1, B)) + 0.05 * rng.standard_normal((T, 12, B))
    force = rng.uniform(0.0, 80.0, (T, 4, B))
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    kp, kd = KP_ROS.copy(), KD_ROS.copy()
    gp = a1.default_gait_params(N)
    # device buffers: the whole run's sensor inputs are uploaded before the first tick
    d_q, d_force, d_mode = eng.dalloc(q.nbytes), eng.dalloc(force.nbytes), eng.dalloc(mode.nbytes)
    _h2d(a1, eng, d_q, q); _h2d(a1, eng, d_force, force); _h2d(a1, eng, d_mode, mode)
    d = a1.DeviceBatch(eng, B)
    d.upload(st)
    d_rz, d_pos, d_lv, d_lvd = eng.dalloc(9 * B * 8), eng.dalloc(3 * B * 8), eng.dalloc(3 * B * 8), eng.dalloc(3 * B * 8)
    _h2d(a1, eng, d_rz, rot_z); _h2d(a1, eng, d_pos, root_pos); _h2d(a1, eng, d_lv, lin_vel); _h2d(a1, eng, d_lvd, lin_vel_d)
    d_gc, d_sp = eng.dalloc(4 * B * 8), eng.dalloc(4 * B * 8)
    _h2d(a1, eng, d_gc, np.zeros((4, B))); _h2d(a1, eng, d_sp, speed)
    d_plan, d_sched, d_trel = eng.dalloc(B * 4), eng.dalloc(N * B * 4), eng.dalloc(12 * B * 8)
    d_jac, d_fk, d_pitch, d_tau = eng.dalloc(36 * B * 8), eng.dalloc(12 * B * 8), eng.dalloc(B * 8), eng.dalloc(12 * B * 8)
    _h2d(a1, eng, d_tau, np.zeros((12, B)))
    sw, warm = eng.swing_alloc(B), eng.warm_alloc(B)
    ext = a1.InputsExt(d_sched.value, None)
    # the CPU chain
    ora = SO.Swing(B)
    ocfg = O.make_config(horizon=N)
    gc0, tau0 = np.zeros((4, B)), np.zeros((12, B))
    Rb = rot.T.reshape(B, 3, 3)
    worst_f = worst_tau = 0.0
    early = 0
    for t in range(T):
        # ---- one tick on the device ----
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, _off(d_q, t * 12 * B * 8), None, d.rot, rho_opt.ctypes.data, rho_fix.ctypes.data, None, d_jac,
                                               None, d.foot, None))
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(gp), d_gc, d_sp, _off(d_mode, t * B * 4), d_lv, d_lvd, d_rz, d.rot, d_pos, d_plan, d_sched,
                                            d_trel, None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, DT, d_gc, d_plan, d_rz, d.foot, d_trel,
                                           _off(d_force, t * 4 * B * 8), d_fk, d.contact, None, None))
        a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, d_pos, d.ref, B, d_pitch))
        a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out), warm, 1))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, d.f_body, d_fk, d_jac, d.contact, km.ctypes.data, tg.ctypes.data, d_tau))
        f, status = d.download()
        con, tau = _d2h(a1, eng, d.contact, B, np.uint32), _d2h(a1, eng, d_tau, (12, B), np.float64)
        fk, e1 = _d2h(a1, eng, d_fk, (12, B), np.float64), _d2h(a1, eng, d.ref, (9, B), np.float64)[1]
        # ---- the same tick from oracle stages ----
        p = np.zeros((B, 4, 3)); J = np.zeros((B, 4, 9))
        for b in range(B):
            for leg in range(4):
                p[b, leg], Jl = O.leg_kinematics(q[t, 3 * leg:3 * leg + 3, b], rho_opt[3 * leg:3 * leg + 3], rho_fix[5 * leg:5 * leg + 5])
                J[b, leg] = Jl.reshape(9)
        fabs = np.einsum("bij,blj->bli", Rb, p).reshape(B, 12).T.copy()
        plan0 = np.zeros(B, dtype=np.uint32); sched0 = np.zeros((N, B), dtype=np.uint32); trel0 = np.zeros((12, B))
        for b in range(B):
            gc0[:, b], plan0[b], sched0[:, b], trel0[:, b], _, _ = O.update_plan(gp, mode[t, b], gc0[:, b], speed[:, b], lin_vel[:, b], lin_vel_d[:, b],
                                                                                 rot_z[:, b], rot[:, b], root_pos[:, b])
        fk0, con0, _, _ = ora.legs(CPS, DT, kp, kd, gc0, plan0, rot_z, fabs, trel0, force[t])
        ref0 = np.ascontiguousarray(ref_in.copy())
        ora.terrain(1, root_pos, ref0)
        fo, info = O.compute_grf_batch_ext(ocfg, O.Batch(x0, rot, fabs, ref0, con0), sched0, None, O.MODE_EXACT, nthreads=O.hardware_threads())
        for b in range(B):
            tau0[:, b] = O.joint_torques(fo[:, b], fk0[:, b], J[b].reshape(36), int(con0[b]), km, tg, tau0[:, b])
        # ---- compare ----
        assert np.array_equal(con, con0), t
        assert (status == a1.STATUS_OPTIMAL).all(), (t, np.bincount(status))
        assert np.abs(e1 - ref0[1]).max() <= 1e-7
        assert (np.abs(fk - fk0) / np.maximum(1.0, np.abs(fk0).max(axis=0))).max() <= 1e-10
        ef = float(np.abs(f - fo).max())
        assert ef <= 1e-4, (t, ef)
        # a force error e moves a stance torque by at most sum_k |J_ka| e; swing torques follow f_kin
        jn = np.abs(J.reshape(B, 4, 3, 3)).sum(axis=2).reshape(B, 12).T
        et = float((np.abs(tau - tau0) - (1e-4 * jn + 1e-8 * np.maximum(1.0, np.abs(tau0)))).max())
        assert et <= 0.0, (t, et)
        worst_f, worst_tau = max(worst_f, ef), max(worst_tau, float(np.abs(tau - tau0).max()))
        early += int(((con & ~plan0) != 0).sum())
    assert early > 0
    d.free()
    for ptr in (d_q, d_force, d_mode, d_rz, d_pos, d_lv, d_lvd, d_gc, d_sp, d_plan, d_sched, d_trel, d_jac, d_fk, d_pitch, d_tau, sw, warm):
        L.a1mpc_device_free(eng.h, ptr)
    print("closed loop B=%d x %d ticks: |f - f_oracle| %.2e N, |tau - tau_oracle| %.2e Nm, %d early-contact legs" % (B, T, worst_f, worst_tau, early))


def test_argument_errors(a1, eng):
    L = a1.lib()
    B = 8
    gp = a1.default_gait_params(N)
    kp, kd = KP_RESET.copy(), KD_RESET.copy()
    h = lambda *s: np.zeros(s)
    gc, rz, fa, tr, ff, pos = h(4, B), h(9, B), h(12, B), h(12, B), h(4, B), h(3, B)
    plan, con, fk = np.zeros(B, dtype=np.uint32), np.zeros(B, dtype=np.uint32), h(12, B)
    sw = eng.swing_alloc(B)
    P = lambda a: a.ctypes.data

    def legs(state=sw, nB=B, gcp=None, rzp=None, fkp=None, conp=None):
        return L.a1mpc_swing_legs_batch(eng.h, nB, C.byref(gp), P(kp), P(kd), state, DT, gcp if gcp is not None else P(gc), P(plan),
                                        rzp if rzp is not None else P(rz), P(fa), P(tr), P(ff), fkp if fkp is not None else P(fk),
                                        conp if conp is not None else P(con), None, None)
    assert legs() == 0
    host_state = np.zeros(B * 921)
    assert legs(state=P(host_state)) == -1 and b"device memory" in L.a1mpc_last_error()
    assert L.a1mpc_swing_init_batch(eng.h, B, P(host_state)) == -1
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, P(host_state), 0, P(pos), None, B, None) == -1
    d_rz = eng.dalloc(9 * B * 8)
    assert legs(rzp=d_rz) == -1 and b"all-host or all-device" in L.a1mpc_last_error()      # mixed sides
    for nb in (0, -3):
        assert legs(nB=nb) == -1
        assert L.a1mpc_swing_init_batch(eng.h, nb, sw) == -1
        assert L.a1mpc_terrain_pitch_batch(eng.h, nb, sw, 0, P(pos), None, B, None) == -1
    for kw in (dict(gcp=C.c_void_p(0)), dict(fkp=C.c_void_p(0)), dict(conp=C.c_void_p(0))):
        rc = L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), P(kp), P(kd), sw, DT, kw.get("gcp", P(gc)), P(plan), P(rz), P(fa), P(tr), P(ff),
                                      kw.get("fkp", P(fk)), kw.get("conp", P(con)), None, None)
        assert rc == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, P(pos), None, B, None) == -1                 # adaptation needs ref
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 0, None, None, B, None) == -1                   # root_pos required
    ref = h(9, B)
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, P(pos), P(ref), B - 1, None) == -1           # ld < B
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, P(pos), d_rz, B, None) == -1                 # mixed sides
    d_kp = eng.dalloc(12 * 8)
    assert L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), d_kp, P(kd), sw, DT, P(gc), P(plan), P(rz), P(fa), P(tr), P(ff), P(fk), P(con), None, None) == -1
    # host path of the terrain call: row 1 only, ld > B respected
    ref = np.full((9, B + 3), 5.0)
    pitch = np.full(B, 9.0)
    assert L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, P(pos), P(ref), B + 3, P(pitch)) == 0
    assert (pitch == 0.0).all() and (ref[1, :B] == 0.0).all() and (ref[1, B:] == 5.0).all() and (np.delete(ref, 1, axis=0) == 5.0).all()
    for p in (sw, d_rz, d_kp):
        L.a1mpc_device_free(eng.h, p)
