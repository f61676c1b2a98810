"""-m gpu: a1mpc_solve_batch_ext and a1mpc_solve_batch_ext_warm on the QPs a closed-loop control tick poses
(tests/sched_tick_scenarios.py, 512 robots x 64 ticks = 32 768 robot-ticks per variant: update_plan's schedules through standstill,
walk / stand switches, early contacts and four-foot crossing steps at all three gait speeds; variants plan, early and terrain),
every QP of every tick against the extended oracle: status OPTIMAL and |f - f*| <= 1e-7 N.  Cold and warm (shift = 1 over the
ticks), on the default handle (pack_ext2_kernel routes all-two-feet schedules to the compacted kernel) and on an
A1MPC_EXT_COMPACT=0 handle (every robot on the general kernel); precision 32 against the optimum of the fp32-rounded inputs
(DESIGN 3).  And the closed loop on device pointers: every stage of the tick as tests/test_gpu_command.py chains them, the solve
given update_plan's schedule on the device (a1mpc_inputs_ext), and for the early variant the swing stage's contacts copied into
schedule step 0.  A failure prints the failing robots' inputs, schedule and tick."""
import ctypes as C
import os

import numpy as np
import pytest

from command_scenarios import DT
from common import obatch
from sched_tick_scenarios import VARIANTS, check_floors, describe, face_census, sched_census, stacked, tick_solve_inputs, variant
from swing_scenarios import KD_ROS, KP_ROS

pytestmark = pytest.mark.gpu

N = 10
B, T, SEED = 512, 64, 43
TOL_CERT = 1e-7     # N: every QP
TOL_LOOP = 1e-4     # N: the device chain's x0 matches the oracle chain's to 1e-8 only, so the loop's forces are held to the suite's gate
ULP = 2.0 ** -23
# counts over the B x T QPs of each variant.  Measured: 22 885 compacted / 9 883 general / 4 507 with a crossing step (plan);
# 17 854 / 14 914 / 9 086 and 452 with a three-foot step (early); 5 376 standstill, 1 024 switches, 9 234 early contacts; oracle
# faces about 31 800 QPs on a friction edge, 10 600-14 000 with a foot-step at the vertex, 2 167-5 644 with a whole foot at the
# vertex, 21 300-22 000 at fz_max
SCHED_FLOORS = dict(compact=15000, general=6000, four=3000, three=200, standstill=3000, switch=800, early=5000)
FACE_FLOORS = dict(edge=20000, vertex=5000, foot0=1000, fzmax=10000)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def D(O):
    """the run and the oracle's optimum (f, info, u_full) of every QP of every variant, stacked over the ticks; generated on the CPU
    once for the module"""
    d = tick_solve_inputs(B, T, SEED, N)
    ocfg = O.make_config(horizon=N)
    d["oracle"], d["stacked"] = {}, {}
    for name in VARIANTS:
        st, sched, normals = d["stacked"][name] = stacked(d, name)
        d["oracle"][name] = O.compute_grf_batch_ext(ocfg, obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
    return d


def _engine(a1, compact=True, **kw):
    if compact:
        return a1.Engine(a1.default_config(horizon=N, **kw))
    os.environ["A1MPC_EXT_COMPACT"] = "0"
    try:
        return a1.Engine(a1.default_config(horizon=N, **kw))
    finally:
        del os.environ["A1MPC_EXT_COMPACT"]


def _check(a1, d, name, what, qps, f, status, tol=TOL_CERT, oracle=None, tol_rel=0.0):
    """QPs `qps` (columns of stacked(d, name)) against the oracle (or `oracle` = (f*, info) of those QPs); returns the largest error"""
    sched = d["stacked"][name][1]
    fo, info = (d["oracle"][name][0][:, qps], d["oracle"][name][1][qps]) if oracle is None else oracle
    none = ~(sched[:, qps] != 0).any(axis=0)
    want = np.where(none, a1.STATUS_NO_CONTACT, a1.STATUS_OPTIMAL)
    err = np.abs(f.astype(np.float64) - fo)
    ef = (err - tol_rel * np.abs(fo)).max(axis=0)
    bad = np.nonzero((status != want) | ~(ef <= tol) | ((info[:, 1] != 1) & ~none))[0]
    assert bad.size == 0, "%s: %d QPs fail (status %s, |f - f*| %s)\n%s" % (
        what, bad.size, status[bad][:8].tolist(), err.max(axis=0)[bad][:8].tolist(), describe(d, name, qps[bad]))
    return float(err.max())


def test_census(D):
    for name in VARIANTS:
        check_floors(name, sched_census(D, name), SCHED_FLOORS if name == "early" else
                     {k: v for k, v in SCHED_FLOORS.items() if k != "three"})
        check_floors(name + " faces", face_census(D, name, D["oracle"][name][2]), FACE_FLOORS)


@pytest.mark.parametrize("compact", [True, False], ids=["routed", "general_only"])
@pytest.mark.parametrize("name", VARIANTS)
def test_cold(a1, D, name, compact):
    """all ticks in one call: the cold solves of different ticks are independent"""
    eng = _engine(a1, compact)
    st, sched, normals = D["stacked"][name]
    f, status, iters = eng.solve_ext(st, sched, normals)
    eng.close()
    kind = "routed" if compact else "general only"
    worst = _check(a1, D, name, "cold %s, %s" % (kind, name), np.arange(B * T), f, status)
    print("%s cold %s: %d QPs, max |f - f*| %.2e N" % (name, kind, B * T, worst))


@pytest.mark.parametrize("compact", [True, False], ids=["routed", "general_only"])
@pytest.mark.parametrize("name", VARIANTS)
def test_warm_over_ticks(a1, D, name, compact):
    eng = _engine(a1, compact)
    warm = eng.warm_alloc(B)
    kind = "routed" if compact else "general only"
    worst, hits = 0.0, []
    for t in range(T):
        st, sched, normals = variant(D, name, t)
        f, status, iters = eng.solve_ext_warm(st, sched, normals, warm, shift=1)
        worst = max(worst, _check(a1, D, name, "warm %s, %s tick %d" % (kind, name, t), t * B + np.arange(B), f, status))
        if t > 0:
            hits.append(((iters % 100) == 0).mean())
    a1.lib().a1mpc_device_free(eng.h, warm)
    eng.close()
    print("%s warm %s: %d QPs, max |f - f*| %.2e N, warm hits %.2f mean" % (name, kind, B * T, worst, np.mean(hits)))
    assert np.mean(hits) > 0.3, hits    # 0.41-0.57 on the emulator: the loop exercises the warm path, not only its cold fall-back


def test_precision32_early(a1, O, D):
    """include/a1mpc.h, precision 32: the optimum of the QP posed by the fp32-rounded inputs, to 1e-4 N + 1 fp32 ulp"""
    eng = _engine(a1, precision=32)
    st, sched, normals = D["stacked"]["early"]
    f, status, iters = eng.solve_ext(st, sched, normals)
    eng.close()
    r = {k: (v if k == "contact" else v.astype(np.float32).astype(np.float64)) for k, v in st.items()}
    fo, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, r), sched, None, O.MODE_EXACT, nthreads=O.hardware_threads())
    assert f.dtype == np.float32
    _check(a1, D, "early", "precision 32", np.arange(B * T), f, status, tol=1e-4, oracle=(fo, info), tol_rel=ULP)


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


@pytest.mark.parametrize("name", ["plan", "early"])
def test_closed_loop_on_device_pointers(a1, O, D, name):
    """tests/test_gpu_command.py's MPC chain on device pointers with the schedule on the device: orientation -> leg kinematics ->
    command -> update_plan (-> d_sched) -> swing legs -> EKF -> terrain pitch -> a1mpc_solve_batch_ext_warm(ext = {d_sched, NULL},
    shift 1) -> joint torques.  For `early` the swing stage's contacts replace schedule step 0; the header has no device-to-device
    copy, so that one row goes through the host.  Against the oracle chain: contacts and modes exact, x0 <= 1e-8, every QP OPTIMAL
    and within 1e-4 N, torques as in the other closed loops."""
    L = a1.lib()
    eng = _engine(a1)
    seqs, speed = D["seqs"], D["speed"]
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    kp, kd = KP_ROS.copy(), KD_ROS.copy()
    rho_opt, rho_fix = np.ascontiguousarray(D["rho_opt"]), np.ascontiguousarray(D["rho_fix"])
    gp = a1.default_gait_params(N)
    cp = a1.default_command_params(a1.VARIANT_GAZEBO)
    ds = {k: eng.dalloc(v.nbytes) for k, v in seqs.items()}
    for k, v in seqs.items():
        _h2d(a1, eng, ds[k], v)
    at = lambda k, t: _off(ds[k], t * seqs[k][0].nbytes)
    d = a1.DeviceBatch(eng, B)
    _h2d(a1, eng, d.x0, np.zeros((12, B)))
    nb = dict(rz=9, ia=3, ig=3, fpr=12, fvr=12, jac=36, kpl=3, des=12, gc=4, sp=4, trel=12, fk=12, tau=12)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    _h2d(a1, eng, dv["gc"], np.zeros((4, B))); _h2d(a1, eng, dv["sp"], speed); _h2d(a1, eng, dv["tau"], np.zeros((12, B)))
    d_mode, d_plan, d_sched, d_est, d_est_status = eng.dalloc(B * 4), eng.dalloc(B * 4), eng.dalloc(N * B * 4), eng.dalloc(B * 4), eng.dalloc(B * 4)
    imu, sw, ekf, warm = eng.imu_alloc(B), eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B)), eng.warm_alloc(B)
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(cp), d.ref, B))
    ext = a1.InputsExt(d_sched.value, None)
    x0p = lambda row: _off(d.x0, row * B * 8)
    tau0 = np.zeros((12, B))
    worst = dict(f=0.0, tau=0.0, x0=0.0)
    for t in range(T):
        a1._check(L.a1mpc_orientation_batch(eng.h, B, at("quat", t), at("gyro", t), at("acc", t), imu, d.rot, dv["rz"], d.x0, B, dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, at("joint_pos", t), at("joint_vel", t), d.rot, rho_opt.ctypes.data, rho_fix.ctypes.data,
                                               dv["fpr"], dv["jac"], dv["fvr"], d.foot, None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, DT, at("cmd", t), x0p(3), B, d_mode, dv["kpl"], d.ref, B, dv["des"], B))
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(gp), dv["gc"], dv["sp"], d_mode, x0p(9), _off(d.ref, 5 * B * 8), dv["rz"], d.rot,
                                            x0p(3), d_plan, d_sched, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, DT, dv["gc"], d_plan, dv["rz"], d.foot,
                                           dv["trel"], at("foot_force", t), dv["fk"], d.contact, None, None))
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], d.rot))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, DT, 1, d_mode, dv["ia"], dv["ig"], d.rot, dv["fpr"], dv["fvr"], at("foot_force", t),
                                               x0p(3), x0p(9), d_est, d_est_status))
        a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, x0p(3), d.ref, B, None))
        if name == "early":
            _h2d(a1, eng, d_sched, _d2h(a1, eng, d.contact, B, np.uint32))      # row 0 of d_sched
        a1._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out), warm, 1))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, d.f_body, dv["fk"], dv["jac"], d.contact, km.ctypes.data, tg.ctypes.data, dv["tau"]))
        f, status = d.download()
        x0 = _d2h(a1, eng, d.x0, (12, B))
        con, mode, tau = _d2h(a1, eng, d.contact, B, np.uint32), _d2h(a1, eng, d_mode, B, np.uint32), _d2h(a1, eng, dv["tau"], (12, B))
        sched = _d2h(a1, eng, d_sched, (N, B), np.uint32)
        # ---- the oracle chain's tick (tests/sched_tick_scenarios.py) ----
        _, sched0, _ = variant(D, name, t)
        fo = D["oracle"][name][0][:, t * B:(t + 1) * B]
        for b in range(B):
            tau0[:, b] = O.joint_torques(fo[:, b], D["fk"][t][:, b], D["jac"][t][:, b], int(D["contact"][t][b]), km, tg, tau0[:, b])
        assert np.array_equal(mode, D["mode"][t]) and np.array_equal(con, D["contact"][t]) and np.array_equal(sched, sched0), t
        ex = float(np.abs(x0 - D["x0"][t]).max())
        assert ex <= 1e-8, (t, ex)
        ef = np.abs(f - fo).max(axis=0)
        bad = np.nonzero((status != a1.STATUS_OPTIMAL) | ~(ef <= TOL_LOOP))[0]
        assert bad.size == 0, "device loop, %s tick %d: %d QPs fail (status %s, |f - f*| %s)\n%s" % (
            name, t, bad.size, status[bad][:8].tolist(), ef[bad][:8].tolist(), describe(D, name, t * B + bad))
        jn = np.abs(D["jac"][t].T.reshape(B, 4, 3, 3)).sum(axis=2).reshape(B, 12).T
        et = float((np.abs(tau - tau0) - (1e-4 * jn + 1e-8 * np.maximum(1.0, np.abs(tau0)))).max())
        assert et <= 0.0, (t, et)
        worst = dict(f=max(worst["f"], float(ef.max())), tau=max(worst["tau"], float(np.abs(tau - tau0).max())), x0=max(worst["x0"], ex))
    d.free()
    for p in list(ds.values()) + list(dv.values()) + [d_mode, d_plan, d_sched, d_est, d_est_status, imu, sw, ekf, warm, cs]:
        L.a1mpc_device_free(eng.h, p)
    eng.close()
    print("device loop %s B=%d x %d ticks: |x0 - x0_oracle| %.2e, |f - f_oracle| %.2e N, |tau - tau_oracle| %.2e Nm" % (
        name, B, T, worst["x0"], worst["f"], worst["tau"]))
