"""ctypes binding of oracle/liba1mpc_swing_oracle.so (swing_oracle.cpp, built by `make -C oracle -f swing.mk`): the oracle of
a1mpc_swing_legs_batch / a1mpc_terrain_pitch_batch.  TEST INFRASTRUCTURE; the product (a1-qp-mpc-controller_b200/) never imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liba1mpc_swing_oracle.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "swing_oracle.cpp")):
            subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "swing.mk", "liba1mpc_swing_oracle.so"])
        L = C.CDLL(_SO)
        L.oracle_swing_new.restype = C.c_void_p
        L.oracle_swing_new.argtypes = [C.c_int]
        L.oracle_swing_free.argtypes = [C.c_void_p]
        L.oracle_swing_legs.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double] + [C.c_void_p] * 12
        L.oracle_terrain_pitch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class Swing:
    """generate_swing_legs_ctrl and compute_grf's terrain adaptation for B robots; the controller state (filters, last positions,
    early contacts) stays inside the oracle object.  Arrays batch-major [F,B] as a1mpc_swing_legs_batch / a1mpc_terrain_pitch_batch."""

    def __init__(self, B):
        L = lib()
        self.L, self.B = L, int(B)
        self.h = C.c_void_p(L.oracle_swing_new(self.B))

    def legs(self, cps, dt, kp, kd, gait_counter, plan_contacts, rot_z, foot_pos_abs, foot_pos_target_rel, foot_force):
        """-> f_kin [12,B], contacts [B], foot_pos_cur [12,B], foot_pos_recent_contact [12,B]"""
        B = self.B
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (kp, kd, gait_counter)]
        pc = np.ascontiguousarray(plan_contacts, dtype=np.uint32)
        b = [np.ascontiguousarray(v, dtype=np.float64) for v in (rot_z, foot_pos_abs, foot_pos_target_rel, foot_force)]
        fk = np.zeros((12, B)); con = np.zeros(B, dtype=np.uint32); cur = np.zeros((12, B)); rc = np.zeros((12, B))
        assert self.L.oracle_swing_legs(self.h, B, C.c_double(cps), C.c_double(dt), *[_ptr(v) for v in a], _ptr(pc), *[_ptr(v) for v in b],
                                        _ptr(fk), _ptr(con), _ptr(cur), _ptr(rc)) == 0
        return fk, con, cur, rc

    def terrain(self, use_terrain_adapt, root_pos, ref=None):
        """-> terrain_pitch [B]; ref [9,B] (if given) gets row 1 when use_terrain_adapt"""
        pos = np.ascontiguousarray(root_pos, dtype=np.float64)
        pitch = np.zeros(self.B)
        assert ref is not None or not use_terrain_adapt
        if ref is not None:
            assert ref.dtype == np.float64 and ref.flags["C_CONTIGUOUS"]
        assert self.L.oracle_terrain_pitch(self.h, self.B, int(use_terrain_adapt), _ptr(pos), _ptr(ref) if ref is not None else None,
                                           ref.shape[1] if ref is not None else 0, _ptr(pitch)) == 0
        return pitch

    def __del__(self):
        try:
            self.L.oracle_swing_free(self.h)
        except Exception:
            pass
