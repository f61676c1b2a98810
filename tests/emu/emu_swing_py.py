"""ctypes binding of the CPU block emulator of a1mpc_swing_legs_batch / a1mpc_terrain_pitch_batch (tests/emu/liba1mpc_emu_swing.so, built
from emu_swing.cpp by swing.mk).  TEST INFRASTRUCTURE, the companion of emu_py.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "swing.mk", "liba1mpc_emu_swing.so"])
        _LIB = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_swing.so"))
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def swing_init(B):
    """a1mpc_swing_init_batch on the emulator: returns the host state [SW_FIELDS, B] (batch-major, as on the device)"""
    L = lib()
    state = np.full((L.emu_swing_fields(), B), np.nan)
    assert L.emu_swing_init(B, _p(state)) == 0
    return state


def swing_legs(state, cps, dt, kp, kd, gait_counter, plan_contacts, rot_z, foot_pos_abs, foot_pos_target_rel, foot_force):
    """a1mpc_swing_legs_batch on the emulator (state updated in place) -> f_kin [12,B], contacts [B], foot_pos_cur, foot_pos_recent_contact"""
    B = state.shape[1]
    assert state.flags["C_CONTIGUOUS"] and state.dtype == np.float64
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (kp, kd, gait_counter)]
    pc = np.ascontiguousarray(plan_contacts, dtype=np.uint32)
    b = [np.ascontiguousarray(v, dtype=np.float64) for v in (rot_z, foot_pos_abs, foot_pos_target_rel, foot_force)]
    fk = np.zeros((12, B)); con = np.zeros(B, dtype=np.uint32); cur = np.zeros((12, B)); rc = np.zeros((12, B))
    assert lib().emu_swing_legs(B, C.c_double(cps), C.c_double(dt), _p(a[0]), _p(a[1]), _p(state), _p(a[2]), _p(pc), *[_p(v) for v in b],
                                _p(fk), _p(con), _p(cur), _p(rc)) == 0
    return fk, con, cur, rc


def terrain_pitch(state, use_terrain_adapt, root_pos, ref):
    """a1mpc_terrain_pitch_batch on the emulator: ref [9,B] row 1 written in place when use_terrain_adapt -> terrain_pitch [B]"""
    B = state.shape[1]
    pos = np.ascontiguousarray(root_pos, dtype=np.float64)
    assert ref.flags["C_CONTIGUOUS"] and ref.dtype == np.float64
    pitch = np.zeros(B)
    assert lib().emu_terrain_pitch(B, _p(state), int(use_terrain_adapt), _p(pos), _p(ref), C.c_size_t(ref.shape[1]), _p(pitch)) == 0
    return pitch
