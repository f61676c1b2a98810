"""ctypes binding of the CPU block emulator of a1mpc_orientation_batch / a1mpc_command_batch (tests/emu/liba1mpc_emu_command.so, built from
emu_command.cpp by command.mk).  TEST INFRASTRUCTURE, the companion of emu_swing_py.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "command.mk", "liba1mpc_emu_command.so"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_command.so"))
        L.emu_imu_init.argtypes = [C.c_int, C.c_void_p]
        L.emu_orientation.argtypes = [C.c_int] + [C.c_void_p] * 8 + [C.c_size_t, C.c_void_p, C.c_void_p]
        L.emu_command_init.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_size_t]
        L.emu_command.argtypes = [C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_size_t, C.c_void_p, C.c_size_t]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _a(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def imu_init(B):
    """a1mpc_imu_init_batch on the emulator: the host state [IM_FIELDS, B]"""
    L = lib()
    state = np.full((L.emu_imu_fields(), B), np.nan)
    assert L.emu_imu_init(B, _p(state)) == 0
    return state


def orientation(quat, gyro, acc=None, imu=None):
    """a1mpc_orientation_batch on the emulator (imu updated in place) -> dict as command_oracle_py.Orientation"""
    q, g = _a(quat), _a(gyro)
    a = _a(acc) if acc is not None else None
    B = q.shape[1]
    o = dict(rot=np.zeros((9, B)), rot_z=np.zeros((9, B)), euler=np.zeros((3, B)), ang_vel=np.zeros((3, B)),
             imu_acc=np.zeros((3, B)) if a is not None else None, imu_ang_vel=np.zeros((3, B)))
    assert lib().emu_orientation(B, _p(q), _p(g), _p(a), _p(imu), _p(o["rot"]), _p(o["rot_z"]), _p(o["euler"]), _p(o["ang_vel"]), B,
                                 _p(o["imu_acc"]), _p(o["imu_ang_vel"])) == 0
    return o


def command_init(B, variant=0, body_height=0.3, hmin=0.1, hmax=0.32, kp_linear=(120.0, 120.0, 500.0), lock=(120.0, 120.0), ref=None):
    """a1mpc_command_init_batch on the emulator: the host state [CM_FIELDS, B]; ref [9,B] gets its reset rows in place"""
    L = lib()
    state = np.full((L.emu_command_fields(), B), np.nan)
    kp, lk = _a(kp_linear), _a(lock)
    assert L.emu_command_init(B, int(variant), body_height, hmin, hmax, _p(kp), _p(lk), _p(state), _p(ref), B) == 0
    return state


def command(state, dt, cmd, root_pos, ref=None):
    """a1mpc_command_batch on the emulator (state, and ref [9,B] when given, updated in place) -> movement_mode, kp_linear [3,B], des [12,B]"""
    B = state.shape[1]
    c, pos = _a(cmd), _a(root_pos)
    if ref is not None:
        assert ref.flags["C_CONTIGUOUS"] and ref.dtype == np.float64
    mode = np.zeros(B, dtype=np.uint32); kp = np.zeros((3, B)); des = np.zeros((12, B))
    assert lib().emu_command(B, C.c_double(dt), _p(state), _p(c), _p(pos), B, _p(mode), _p(kp), _p(ref), B, _p(des), B) == 0
    return mode, kp, des
