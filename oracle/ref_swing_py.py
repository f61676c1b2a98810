"""ctypes binding of oracle/_ref/libref_swing.so: the REFERENCE'S OWN A1RobotControl.cpp (and the sources it links) compiled unmodified
against the header stand-ins of oracle/ref_shim/, with the multi-tick driver ref_swing_wrap.cpp (`make -C oracle -f swing.mk ref`).
TEST INFRASTRUCTURE.

Exists only where the reference sources were present when that build ran.  No GPU test may depend on it: tests use
tests/golden/swing_v1.npz (tests/golden/make_swing_golden.py) and call `available()` before touching anything here."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libref_swing.so")
_LIB = None


def available():
    return os.path.exists(_SO)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(_SO)
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a(v):
    return np.ascontiguousarray(v, dtype=np.float64).reshape(-1)


def swing_ticks(kp, kd, gait_counter_speed, movement_mode, lin_vel, lin_vel_d, root_pos, rot_z, rot, foot_pos_abs, foot_force, use_terrain_adapt=1,
                dt=0.0025):
    """T ticks of update_plan -> generate_swing_legs_ctrl -> compute_grf (MPC branch, QP answered by zeros) on ONE reference controller.
    Inputs tick-major: movement_mode [T], lin_vel / lin_vel_d / root_pos [T,3], rot_z / rot [T,9], foot_pos_abs [T,12], foot_force [T,4].
    Returns dict of per-tick records: gait_counter [T,4], plan_contacts [T], contacts [T], foot_pos_target_rel, f_kin, foot_pos_cur,
    foot_pos_recent_contact [T,12], root_euler_d1 [T], terrain_pitch [T]."""
    L = lib()
    mm = np.ascontiguousarray(movement_mode, dtype=np.int32)
    T = mm.shape[0]
    a = [_a(v) for v in (kp, kd, gait_counter_speed, lin_vel, lin_vel_d, root_pos, rot_z, rot, foot_pos_abs, foot_force)]
    assert a[0].size == 12 and a[1].size == 12 and a[2].size == 4 and a[3].size == 3 * T and a[8].size == 12 * T and a[9].size == 4 * T
    o = dict(gait_counter=np.zeros((T, 4)), plan_contacts=np.zeros(T, dtype=np.uint32), contacts=np.zeros(T, dtype=np.uint32),
             foot_pos_target_rel=np.zeros((T, 12)), f_kin=np.zeros((T, 12)), foot_pos_cur=np.zeros((T, 12)), foot_pos_recent_contact=np.zeros((T, 12)),
             root_euler_d1=np.zeros(T), terrain_pitch=np.zeros(T))
    rc = L.ref_swing_ticks(int(T), int(use_terrain_adapt), C.c_double(dt), _p(a[0]), _p(a[1]), _p(a[2]), _p(mm), *[_p(v) for v in a[3:]],
                           *[_p(o[k]) for k in ("gait_counter", "plan_contacts", "contacts", "foot_pos_target_rel", "f_kin", "foot_pos_cur",
                                                "foot_pos_recent_contact", "root_euler_d1", "terrain_pitch")])
    assert rc == 0
    return o
