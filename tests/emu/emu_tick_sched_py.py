"""ctypes binding of the CPU block emulator of the scheduled tick's front kernel and the staged kernels it fuses
(tests/emu/liba1mpc_emu_tick_sched.so, built from emu_tick_sched.cpp by tick_sched.mk).  TEST INFRASTRUCTURE, the companion of
emu_tick_py.py.  Every array is a contiguous float64 / uint32 numpy array, dense [rows][B], updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

from emu_tick_py import gait17

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "tick_sched.mk", "all"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_tick_sched.so"))
        L.emu_front_sched_staged.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_double, C.c_int] + [C.c_void_p] * 20
        L.emu_front_sched_fused.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_double, C.c_int] + [C.c_void_p] * 18
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def front_sched(fused, B, tp, dt, N, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts,
                sched, plan=None, trel=None):
    """kinematics + update_plan with the schedule sched [N][B] + swing legs: tick_front_sched (fused) or the three staged kernels with row 0
    of the schedule overwritten by the swing stage's contacts (plan [B], trel [12][B]: their hand-over)"""
    L = lib()
    arr = lambda v: np.ascontiguousarray(v, dtype=np.float64)
    pars = [arr(tp.rho_opt), arr(tp.rho_fix), gait17(tp.gait), arr(tp.kp_foot), arr(tp.kd_foot)]
    io = [joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts, sched]
    if fused:
        rc = L.emu_front_sched_fused(B, *(_p(x) for x in pars), dt, N, *(_p(x) for x in io))
    else:
        rc = L.emu_front_sched_staged(B, *(_p(x) for x in pars), dt, N, *(_p(x) for x in io + [plan, trel]))
    assert rc == 0


def swing_fields():
    return lib().emu_sched_swing_fields()
