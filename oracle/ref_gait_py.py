"""ctypes binding of oracle/_ref/libref_gait.so: the REFERENCE'S OWN A1RobotControl.cpp (and the sources it links) compiled unmodified
against the header stand-ins of oracle/ref_shim/, with the per-robot-gait driver ref_gait_wrap.cpp (`make -C oracle -f gait.mk ref`).
TEST INFRASTRUCTURE.  Exists only where the reference sources were present when that build ran: call `available()` first."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libref_gait.so")
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


def gait_ticks(row, kp, kd, gait_counter_speed, movement_mode, lin_vel, lin_vel_d, root_pos, rot_z, rot, foot_pos_abs, foot_force, dt=0.0025):
    """T ticks of update_plan -> generate_swing_legs_ctrl on ONE reference controller with the gait row `row` [6].  Inputs tick-major as
    ref_swing_py.swing_ticks.  Returns dict of per-tick records: gait_counter [T,4], plan_contacts [T], contacts [T], foot_pos_target_rel,
    f_kin, foot_pos_cur, foot_pos_recent_contact [T,12]."""
    L = lib()
    mm = np.ascontiguousarray(movement_mode, dtype=np.int32)
    T = mm.shape[0]
    a = [_a(v) for v in (row, kp, kd, gait_counter_speed, lin_vel, lin_vel_d, root_pos, rot_z, rot, foot_pos_abs, foot_force)]
    assert a[0].size == 6 and a[1].size == 12 and a[3].size == 4 and a[4].size == 3 * T and a[9].size == 12 * T and a[10].size == 4 * T
    o = dict(gait_counter=np.zeros((T, 4)), plan_contacts=np.zeros(T, dtype=np.uint32), contacts=np.zeros(T, dtype=np.uint32),
             foot_pos_target_rel=np.zeros((T, 12)), f_kin=np.zeros((T, 12)), foot_pos_cur=np.zeros((T, 12)), foot_pos_recent_contact=np.zeros((T, 12)))
    rc = L.ref_gait_ticks(int(T), _p(a[0]), C.c_double(dt), _p(a[1]), _p(a[2]), _p(a[3]), _p(mm), *[_p(v) for v in a[4:]],
                          *[_p(o[k]) for k in ("gait_counter", "plan_contacts", "contacts", "foot_pos_target_rel", "f_kin", "foot_pos_cur",
                                               "foot_pos_recent_contact")])
    assert rc == 0
    return o
