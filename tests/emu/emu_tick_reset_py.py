"""ctypes binding of the CPU block emulator of the tick's masked reset kernels (tests/emu/liba1mpc_emu_tick_reset.so, built from
emu_tick_reset.cpp by tick_reset.mk).  TEST INFRASTRUCTURE, the companion of emu_tick_py.py.  Every array is a contiguous float64 / uint32 /
uint8 numpy array, dense [rows][B] (the EKF state [B][342]), updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "tick_reset.mk", "all"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_tick_reset.so"))
        L.emu_reset_sizes.argtypes = [C.c_void_p]
        L.emu_tick_reset_robots.argtypes = [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_void_p]
        L.emu_init_kernels.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 7
        L.emu_ekf_init.argtypes = [C.c_int] + [C.c_void_p] * 3
        L.emu_ekf_init_pending.argtypes = [C.c_int] + [C.c_void_p] * 5
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32, np.uint8), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def sizes():
    """dict of the per-robot state sizes: imu, cmd, swing, ekf (doubles) and warm_hdr (words)"""
    out = np.zeros(5, dtype=np.int32)
    lib().emu_reset_sizes(out.ctypes.data_as(C.c_void_p))
    return dict(zip(("imu", "cmd", "swing", "ekf", "warm_hdr"), (int(v) for v in out)))


def _cparams(cp):
    return (np.array([cp.body_height, cp.body_height_min, cp.body_height_max]), np.array(cp.kp_linear, dtype=np.float64),
            np.array(cp.kp_linear_lock, dtype=np.float64))


def reset_robots(B, mask, cp, x0, gc, tau, imu, cmd, ref, swing, warm, warm_words, pending):
    """tick_reset_robots_kernel with the start values of a1mpc_command_params cp"""
    hp, kp, lock = _cparams(cp)
    assert lib().emu_tick_reset_robots(B, _p(mask), cp.variant, _p(hp), _p(kp), _p(lock), *(_p(a) for a in (x0, gc, tau, imu, cmd, ref, swing, warm)),
                                       warm_words, _p(pending)) == 0


def init_kernels(B, cp, imu, cmd, ref, swing):
    """imu_init_kernel (imu may be None), command_init_kernel and swing_init_kernel over the whole batch"""
    hp, kp, lock = _cparams(cp)
    assert lib().emu_init_kernels(B, cp.variant, _p(hp), _p(kp), _p(lock), *(_p(a) for a in (imu, cmd, ref, swing))) == 0


def ekf_init(B, ekf, fpr, rot):
    assert lib().emu_ekf_init(B, _p(ekf), _p(fpr), _p(rot)) == 0


def ekf_init_pending(B, pending, ekf, fpr, rot, x0):
    assert lib().emu_ekf_init_pending(B, _p(pending), _p(ekf), _p(fpr), _p(rot), _p(x0)) == 0
