"""ctypes binding of the CPU block emulator of the per-robot gait kernels (tests/emu/liba1mpc_emu_gait.so, built from emu_gait.cpp by
gait.mk).  TEST INFRASTRUCTURE.  Every array is a contiguous float64 / uint32 numpy array, dense [rows][B], updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

from emu_tick_py import gait17

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
PLAIN, TWIN, STAGED = 0, 1, 2


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "gait.mk", "all"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_gait.so"))
        L.emu_gait_front.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_double, C.c_int] + [C.c_void_p] * 21
        L.emu_gait_update_plan.argtypes = [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 14
        L.emu_gait_swing_legs.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_double] + [C.c_void_p] * 12
        L.emu_gait_check.argtypes = [C.c_int, C.c_void_p]
        L.emu_gait_check.restype = C.c_ulonglong
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def front(kind, B, tp, dt, N, gait, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts,
          sched=None, plan=None, trel=None):
    """the tick's front stage: PLAIN (tick_front_b / _sched), TWIN (their gait twins) or STAGED (the staged gait kernels)"""
    arr = lambda v: np.ascontiguousarray(v, dtype=np.float64)
    pars = [arr(tp.rho_opt), arr(tp.rho_fix), gait17(tp.gait), arr(tp.kp_foot), arr(tp.kd_foot)]
    io = [gait, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts, sched, plan, trel]
    assert lib().emu_gait_front(kind, B, *(_p(x) for x in pars), dt, N, *(_p(x) for x in io)) == 0


def update_plan(gp, gait, gc, gcs, mode, lv, lvd, rz, rot, pos, plan, sched, t_rel, t_abs, t_world):
    B = gc.shape[1]
    io = [gait, gc, gcs, mode, lv, lvd, rz, rot, pos, plan, sched, t_rel, t_abs, t_world]
    assert lib().emu_gait_update_plan(B, _p(gait17(gp)), int(gp.horizon), *(_p(x) for x in io)) == 0


def swing_legs(gp, kp, kd, dt, gait, swing, gc, plan, rz, fpa, tgt, ff, fkin, contacts, cur, rc):
    B = gc.shape[1]
    io = [gait, swing, gc, plan, rz, fpa, tgt, ff, fkin, contacts, cur, rc]
    assert lib().emu_gait_swing_legs(B, _p(gait17(gp)), _p(np.ascontiguousarray(kp, dtype=np.float64)), _p(np.ascontiguousarray(kd, dtype=np.float64)),
                                     dt, *(_p(x) for x in io)) == 0


def check(gait):
    """gait_check_kernel -> None, or (robot, rule) of the first bad row"""
    g = np.ascontiguousarray(gait, dtype=np.float64)
    bad = lib().emu_gait_check(g.shape[1], _p(g))
    return None if bad == (1 << 64) - 1 else (bad >> 2, bad & 3)


def swing_fields():
    return lib().emu_gait_swing_fields()
