"""ctypes binding of the CPU block emulator of a1mpc_stance_qp_batch_ext and a1mpc_surface_normals_batch
(tests/emu/liba1mpc_emu_stance_terrain.so, built from emu_stance_terrain.cpp by stance_terrain.mk).  TEST INFRASTRUCTURE, the companion of
emu_stance_py.py and emu_terrain_normals_py.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "stance_terrain.mk", "liba1mpc_emu_stance_terrain.so"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_stance_terrain.so"))
        L.emu_st_stance_qp.argtypes = [C.c_int, C.c_size_t] + [C.c_void_p] * 8 + [C.c_double] + [C.c_void_p] * 4 + [C.c_int]
        L.emu_st_surface_normals.argtypes = [C.c_int] + [C.c_void_p] * 3
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def stance_qp(x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, mass, normals=None, order=0):
    """a1mpc_stance_qp_batch_ext on the emulator (normals [12,B]; None: a1mpc_stance_qp_batch), batch-major host arrays (ld = B) ->
    f_body [12,B], status [B], root_acc [6,B]"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x0, rot, rot_z, foot)]
    contact = np.ascontiguousarray(contact, dtype=np.uint32)
    d, kpl = np.ascontiguousarray(des, dtype=np.float64), np.ascontiguousarray(kp_linear, dtype=np.float64)
    gains = np.ascontiguousarray(np.concatenate([kd_linear, kp_angular, kd_angular]), dtype=np.float64)
    nrm = np.ascontiguousarray(normals, dtype=np.float64) if normals is not None else None
    B = contact.shape[0]
    f = np.full((12, B), np.nan); status = np.full(B, -7, dtype=np.int32); acc = np.full((6, B), np.nan)
    assert lib().emu_st_stance_qp(B, B, *[_p(v) for v in a], _p(contact), _p(d), _p(kpl), _p(gains), mass, _p(nrm), _p(f), _p(status), _p(acc),
                                  int(order)) == 0
    return f, status, acc


def surface_normals(state, root_pos):
    """surface_normals_kernel: state [SW_FIELDS,B] (read only), root_pos [3,B] -> normals [12,B]"""
    assert state.flags.c_contiguous and state.dtype == np.float64
    B = state.shape[1]
    pos = np.ascontiguousarray(root_pos, dtype=np.float64)
    normals = np.full((12, B), np.nan)
    assert lib().emu_st_surface_normals(B, _p(state), _p(pos), _p(normals)) == 0
    return normals
