"""ctypes binding of oracle/liba1mpc_stance_terrain_oracle.so (stance_terrain_oracle.cpp, built by `make -C oracle -f stance_terrain.mk`):
compute_grf's 12-force QP (oracle_py.grf_qp_single) with each foot's friction pyramid in its terrain frame, the exact solve, one robot or
a batch on host threads.  TEST INFRASTRUCTURE; the product (a1-qp-mpc-controller_b200/) never imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liba1mpc_stance_terrain_oracle.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "stance_terrain_oracle.cpp")):
            subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "stance_terrain.mk", "liba1mpc_stance_terrain_oracle.so"])
        L = C.CDLL(_SO)
        L.oracle_grf_qp_single_ext.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.oracle_grf_qp_batch_ext.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def grf_qp_single_ext(root_acc, rot_z, rot, foot, contact, normals12):
    """one robot: f_body [12], info [8] (iters, verified, kkt_stat, kkt_prim, kkt_dual, rounds)"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (root_acc, rot_z, rot, foot, normals12)]
    f = np.zeros(12); info = np.zeros(8)
    assert lib().oracle_grf_qp_single_ext(_ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), int(contact), _ptr(a[4]), 0, _ptr(f), _ptr(info)) == 0
    return f, info


def grf_qp_batch_ext(root_acc, rot_z, rot, foot, contact, normals, nthreads=None):
    """batch-major [6,B], [9,B], [9,B], [12,B], [B], [12,B] -> f_body [12,B], info [B,8]; a robot without a stance foot: zero forces,
    info[1] = 1"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (root_acc, rot_z, rot, foot, normals)]
    c = np.ascontiguousarray(contact, dtype=np.uint32)
    B = c.shape[0]
    assert [v.shape for v in a] == [(6, B), (9, B), (9, B), (12, B), (12, B)]
    f = np.zeros((12, B)); info = np.zeros((B, 8))
    nthreads = nthreads or os.cpu_count() or 1
    lib().oracle_grf_qp_batch_ext(B, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), _ptr(c), _ptr(a[4]), int(nthreads), _ptr(f), _ptr(info))
    return f, info
