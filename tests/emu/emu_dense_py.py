"""ctypes binding of the CPU block emulator of a1mpc_solve_dense_batch and a1mpc_grf_qp_batch (tests/emu/liba1mpc_emu_dense.so, built
from emu_dense.cpp by dense.mk).  TEST INFRASTRUCTURE, the companion of emu_py.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(_HERE)), "a1-qp-mpc-controller_b200"))
import a1mpc  # noqa: E402  (struct definitions only; the emulator never touches liba1mpc.so)

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "dense.mk", "liba1mpc_emu_dense.so"])
        _LIB = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_dense.so"))
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def solve_dense(cfg, H, g, contact, order=0, max_blocks=0, nthreads=1):
    """a1mpc_solve_dense_batch on the emulator, N = 10 or 20: H [B,n,n], g [B,n], contact [B] -> u [B,n], status [B].  u and status start
    as NaN and -7, so a QP the solve never writes shows.  max_blocks > 0 caps each class's grid, so a block solves several QPs in turn
    as a device CTA does; 0 runs one block per QP.  nthreads: host threads over the blocks of a class (the result does not depend on it)"""
    H = np.ascontiguousarray(H, dtype=np.float64); g = np.ascontiguousarray(g, dtype=np.float64)
    contact = np.ascontiguousarray(contact, dtype=np.uint32)
    B, n = g.shape
    u = np.full((B, n), np.nan); status = np.full(B, -7, dtype=np.int32)
    assert lib().emu_dense_solve(C.byref(cfg), B, _p(H), _p(g), _p(contact), _p(u), _p(status), int(order), int(max_blocks), int(nthreads)) == 0
    return u, status


def grf_qp(root_acc, rot_z, rot, foot, contact, order=0, max_blocks=0):
    """a1mpc_grf_qp_batch on the emulator: root_acc [B,6], rot_z/rot [B,9], foot [B,12], contact [B] -> f_body [B,12], status [B]"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (root_acc, rot_z, rot, foot)]
    contact = np.ascontiguousarray(contact, dtype=np.uint32)
    B = contact.shape[0]
    f = np.full((B, 12), np.nan); status = np.full(B, -7, dtype=np.int32)
    assert lib().emu_dense_grf_qp(B, _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(contact), _p(f), _p(status), int(order), int(max_blocks)) == 0
    return f, status
