"""ctypes binding of the CPU block emulator of the terrain stage with normals (tests/emu/liba1mpc_emu_terrain_normals.so, built from
emu_terrain_normals.cpp by terrain_normals.mk).  TEST INFRASTRUCTURE, the companion of emu_swing_py.py.  Every array is a contiguous
float64 / uint32 numpy array, dense [rows][B]; the swing state [SW_FIELDS][B] is updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "terrain_normals.mk", "all"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_terrain_normals.so"))
        L.emu_tn_swing_init.argtypes = [C.c_int, C.c_void_p]
        L.emu_tn_swing_legs.argtypes = [C.c_int, C.c_double, C.c_double] + [C.c_void_p] * 12
        L.emu_tn_terrain_pitch.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.emu_tn_terrain_normals.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t] + [C.c_void_p] * 4 + [C.c_int]
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def swing_init(B):
    """swing_init_kernel: the zero state [SW_FIELDS, B]"""
    state = np.full((lib().emu_tn_swing_fields(), B), np.nan)
    assert lib().emu_tn_swing_init(B, _p(state)) == 0
    return state


def swing_legs(state, cps, dt, kp, kd, gait_counter, plan_contacts, rot_z, foot_pos_abs, foot_pos_target_rel, foot_force):
    """swing_legs_kernel (state in place) -> contacts [B], foot_pos_recent_contact [12,B]"""
    B = state.shape[1]
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    fk, con, rc = np.zeros((12, B)), np.zeros(B, dtype=np.uint32), np.zeros((12, B))
    assert lib().emu_tn_swing_legs(B, cps, dt, _p(f(kp)), _p(f(kd)), _p(state), _p(f(gait_counter)), _p(np.ascontiguousarray(plan_contacts, dtype=np.uint32)),
                                   _p(f(rot_z)), _p(f(foot_pos_abs)), _p(f(foot_pos_target_rel)), _p(f(foot_force)), _p(fk), _p(con), _p(rc)) == 0
    return con, rc


def terrain_pitch(state, adapt, root_pos, ref):
    """terrain_pitch_kernel: ref [9,B] row 1 in place when adapt -> terrain_pitch [B]"""
    B = state.shape[1]
    pitch = np.zeros(B)
    assert lib().emu_tn_terrain_pitch(B, _p(state), int(adapt), _p(np.ascontiguousarray(root_pos, dtype=np.float64)), _p(ref), ref.shape[1],
                                      _p(pitch)) == 0
    return pitch


def terrain_normals(state, adapt, root_pos, ref, contacts=None, N=0):
    """terrain_normals_kernel: ref [9,B] row 1 in place when adapt -> (terrain_pitch [B], normals [12,B], sched [N,B] or None); with
    contacts the kernel writes them into all N rows of sched, the tick's held pattern"""
    B = state.shape[1]
    pitch, normals = np.zeros(B), np.full((12, B), np.nan)
    sched = np.zeros((N, B), dtype=np.uint32) if contacts is not None else None
    c = np.ascontiguousarray(contacts, dtype=np.uint32) if contacts is not None else None
    assert lib().emu_tn_terrain_normals(B, _p(state), int(adapt), _p(np.ascontiguousarray(root_pos, dtype=np.float64)), _p(ref), ref.shape[1],
                                        _p(pitch), _p(normals), _p(c), _p(sched), N) == 0
    return pitch, normals, sched
