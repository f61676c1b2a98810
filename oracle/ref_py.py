"""ctypes binding of oracle/_ref/libref_mpc.so: the REFERENCE'S OWN sources (ConvexMpc.cpp, A1RobotControl.cpp, A1BasicEKF.cpp,
utils/Utils.cpp) compiled unmodified against the header stand-ins of oracle/ref_shim/ (`make -C oracle ref`).  TEST INFRASTRUCTURE.

Exists only where the reference sources were present when `make -C oracle ref` ran.  No GPU test may depend on it: tests use tests/golden/convexmpc_v1.npz (tools: tests/golden/make_ref_golden.py) and call `available()` before
touching anything here.  The QP that the reference hands to OsqpEigen is solved by the oracle's OSQP-algorithm restatement
(`solver="tight"`: eps 1e-11; "default": OSQP defaults) -- OSQP itself is third party and absent.
"""
import ctypes as C
import os

import numpy as np

from . import oracle_py as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libref_mpc.so")
_LIB = None
N = 10  # A1Params.h:26, compile-time in the reference


def available():
    return os.path.exists(_SO)


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _a(v, n=None):
    a = np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
    assert n is None or a.size == n, (a.size, n)
    return a


def lib(solver="tight"):
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(_SO)
        _LIB.ref_ekf_new.restype = C.c_void_p
        assert _LIB.ref_plan_horizon() == N
    ol = O.lib()
    fn = {"tight": ol.oracle_qp_hook_osqp_tight, "default": ol.oracle_qp_hook_osqp_default}[solver]
    _LIB.ref_set_qp_solver(C.cast(fn, C.c_void_p))
    return _LIB


def last_qp():
    """the problem of the latest OsqpEigen::Solver::solve(): P [n,n] (symmetric completion of the upper triangle the reference
    hands over), q, A [m,n], l, u"""
    L = lib()
    n, m = C.c_int(), C.c_int()
    L.ref_last_qp_dims(C.byref(n), C.byref(m))
    n, m = n.value, m.value
    P = np.zeros((n, n)); q = np.zeros(n); A = np.zeros((m, n)); l = np.zeros(m); u = np.zeros(m)
    assert L.ref_last_qp(_p(P), _p(q), _p(A), _p(l), _p(u)) == 0
    return P, q, A, l, u


def convexmpc(q, r, euler, mass, inertia, rot, foot, dt, mpc_states, mpc_states_d, contact, foot_shift=None):
    """ConvexMpc driven as compute_grf drives it (foot_shift None) or as test/test_mpc.cpp does (feet move by -foot_shift per step).
    Returns dict of row-major arrays: A_qp, B_qp, H, g, Ac, lb, ub, B_d_list, A_d."""
    L = lib()
    o = dict(A_qp=np.zeros((13 * N, 13)), B_qp=np.zeros((13 * N, 12 * N)), H=np.zeros((12 * N, 12 * N)), g=np.zeros(12 * N),
             Ac=np.zeros((20 * N, 12 * N)), lb=np.zeros(20 * N), ub=np.zeros(20 * N), B_d_list=np.zeros((13 * N, 12)), A_d=np.zeros((13, 13)))
    fs = _a(foot_shift, 3) if foot_shift is not None else None
    a = [_a(q, 13), _a(r, 12), _a(euler, 3), _a(inertia, 9), _a(rot, 9), _a(foot, 12), _a(mpc_states, 13), _a(mpc_states_d, 13 * N)]
    rc = L.ref_convexmpc(_p(a[0]), _p(a[1]), _p(a[2]), C.c_double(mass), _p(a[3]), _p(a[4]), _p(a[5]), _p(fs), C.c_double(dt), _p(a[6]), _p(a[7]),
                         C.c_uint32(int(contact)), _p(o["A_qp"]), _p(o["B_qp"]), _p(o["H"]), _p(o["g"]), _p(o["Ac"]), _p(o["lb"]), _p(o["ub"]),
                         _p(o["B_d_list"]), _p(o["A_d"]))
    assert rc == 0
    return o


def compute_grf(cfg, x0, rot, foot, ref, contact, control_type=1, ticks=1, solver="tight", use_terrain_adapt=0, rot_z=None, root_pos_d_xy=(0.0, 0.0),
                yaw_d=0.0, gains=None):
    """A1RobotControl::compute_grf on one robot given in the a1mpc_inputs layout (x0[12], rot[9], foot[12], ref[9], contact mask).
    Returns dict(f_body[12], mpc_states[13], mpc_states_d[130], root_lin_vel_d_world[3], root_euler_d[3], qp=(P,q,A,l,u))."""
    L = lib(solver)
    ref = _a(ref, 9)
    # ref: root_euler_d[0], root_euler_d[1], root_ang_vel_d(3), root_lin_vel_d(3), root_pos_d[2]  (include/a1mpc.h)
    ref12 = np.array([ref[0], ref[1], yaw_d, root_pos_d_xy[0], root_pos_d_xy[1], ref[8], ref[5], ref[6], ref[7], ref[2], ref[3], ref[4]])
    f = np.zeros(12); ms = np.zeros(13); msd = np.zeros(13 * N); vw = np.zeros(3); ed = np.zeros(3)
    a = [_a(cfg.q[:], 13), _a(cfg.r[:], 12), _a(cfg.inertia[:], 9), _a(x0, 12), _a(rot, 9), _a(foot, 12)]
    rz = _a(rot_z, 9) if rot_z is not None else None
    gn = _a(gains, 12) if gains is not None else None
    rc = L.ref_compute_grf(int(control_type), int(use_terrain_adapt), C.c_double(cfg.dt), int(ticks), _p(a[0]), _p(a[1]), C.c_double(cfg.mass), _p(a[2]),
                           _p(a[3]), _p(a[4]), _p(rz), _p(a[5]), C.c_uint32(int(contact)), _p(ref12), _p(gn), _p(f), _p(ms), _p(msd), _p(vw), _p(ed))
    assert rc == 0
    return dict(f_body=f, mpc_states=ms, mpc_states_d=msd, root_lin_vel_d_world=vw, root_euler_d=ed, qp=last_qp())


def joint_torques(f_grf, f_kin, jac, contact, km_foot, torques_gravity, tau_prev=None):
    L = lib()
    tau = np.zeros(12)
    a = [_a(f_grf, 12), _a(f_kin, 12), _a(jac, 36), _a(km_foot, 3), _a(torques_gravity, 12)]
    tp = _a(tau_prev, 12) if tau_prev is not None else None
    L.ref_joint_torques(_p(a[0]), _p(a[1]), _p(a[2]), C.c_uint32(int(contact)), _p(a[3]), _p(a[4]), _p(tp), _p(tau))
    return tau


def update_plan(counter_per_gait, counter_per_swing, control_dt, default_foot_pos, movement_mode, gait_counter, gait_counter_speed, lin_vel, lin_vel_d,
                rot_z, rot, root_pos, dt=0.0025):
    L = lib()
    gc = np.array(gait_counter, dtype=np.float64)
    a = [_a(default_foot_pos, 12), _a(gait_counter_speed, 4), _a(lin_vel, 3), _a(lin_vel_d, 3), _a(rot_z, 9), _a(rot, 9), _a(root_pos, 3)]
    plan = C.c_uint32(); trel = np.zeros(12); tabs = np.zeros(12); tw = np.zeros(12)
    L.ref_update_plan(C.c_double(counter_per_gait), C.c_double(counter_per_swing), C.c_double(control_dt), _p(a[0]), int(movement_mode), _p(gc), _p(a[1]),
                      _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), _p(a[6]), C.c_double(dt), C.byref(plan), _p(trel), _p(tabs), _p(tw))
    return gc, int(plan.value), trel, tabs, tw


class Ekf:
    """A1BasicEKF, the filter state stays inside the reference object"""

    def __init__(self, assume_flat_ground=True):
        self.L = lib()
        self.h = C.c_void_p(self.L.ref_ekf_new(int(assume_flat_ground)))

    def init(self, foot_pos_rel, rot):
        x = np.zeros(18); P = np.zeros((18, 18))
        a = [_a(foot_pos_rel, 12), _a(rot, 9)]
        self.L.ref_ekf_init(self.h, _p(a[0]), _p(a[1]), _p(x), _p(P))
        return x, P

    def update(self, dt, movement_mode, imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel, foot_force):
        x = np.zeros(18); P = np.zeros((18, 18)); pos = np.zeros(3); vel = np.zeros(3); ec = C.c_uint32()
        a = [_a(imu_acc, 3), _a(imu_ang_vel, 3), _a(rot, 9), _a(foot_pos_rel, 12), _a(foot_vel_rel, 12), _a(foot_force, 4)]
        self.L.ref_ekf_update(self.h, C.c_double(dt), int(movement_mode), *[_p(v) for v in a], _p(x), _p(P), _p(pos), _p(vel), C.byref(ec))
        return x, P, pos, vel, int(ec.value)

    def __del__(self):
        try:
            self.L.ref_ekf_free(self.h)
        except Exception:
            pass
