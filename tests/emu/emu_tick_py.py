"""ctypes binding of the CPU block emulator of the fused tick kernels and the staged kernels they fuse (tests/emu/liba1mpc_emu_tick_{a,b}.so,
built from emu_tick.cpp by tick.mk).  TEST INFRASTRUCTURE, the companion of emu_command_py.py and emu_swing_py.py.  Every array is a
contiguous float64 / uint32 numpy array, dense [rows][B], updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = None


def libs():
    global _LIBS
    if _LIBS is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "tick.mk", "all"])
        a = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_tick_a.so"))
        b = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_tick_b.so"))
        for f in (a.emu_front_a_staged, a.emu_front_a_fused):
            f.argtypes = [C.c_int, C.c_double] + [C.c_void_p] * 15
        b.emu_front_b_staged.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_double] + [C.c_void_p] * 19
        b.emu_front_b_fused.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_double] + [C.c_void_p] * 17
        _LIBS = (a, b)
    return _LIBS


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def front_a(fused, B, dt, quat, gyro, acc, imu, rot, rot_z, x0, imu_acc, imu_ang_vel, cmd_state, cmd, mode, kp, ref, des):
    """orientation + command: tick_front_a (fused) or orientation_kernel then command_kernel"""
    L = libs()[0]
    f = L.emu_front_a_fused if fused else L.emu_front_a_staged
    assert f(B, dt, *(_p(x) for x in (quat, gyro, acc, imu, rot, rot_z, x0, imu_acc, imu_ang_vel, cmd_state, cmd, mode, kp, ref, des))) == 0


def gait17(gp):
    return np.array([gp.counter_per_gait, gp.counter_per_swing, gp.control_dt] + list(gp.default_foot_pos) +
                    [gp.foot_delta_x_limit, gp.foot_delta_y_limit])


def front_b(fused, B, tp, dt, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts,
            plan=None, trel=None):
    """kinematics + update_plan + swing legs: tick_front_b (fused) or the three staged kernels (plan [B], trel [12][B]: their hand-over)"""
    L = libs()[1]
    arr = lambda v: np.ascontiguousarray(v, dtype=np.float64)
    pars = [arr(tp.rho_opt), arr(tp.rho_fix), gait17(tp.gait), arr(tp.kp_foot), arr(tp.kd_foot)]
    io = [joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts]
    if fused:
        rc = L.emu_front_b_fused(B, *(_p(x) for x in pars), dt, *(_p(x) for x in io))
    else:
        rc = L.emu_front_b_staged(B, *(_p(x) for x in pars), dt, *(_p(x) for x in io + [plan, trel]))
    assert rc == 0


def swing_fields():
    return libs()[1].emu_swing_fields()
