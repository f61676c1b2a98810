"""ctypes binding of the CPU block emulator of a1mpc_solve_batch_ext_warm (tests/emu/liba1mpc_emu_ext_warm.so, built from
emu_ext_warm.cpp by ext_warm.mk).  TEST INFRASTRUCTURE, the companion of emu_py.py."""
import ctypes as C
import os
import subprocess

import numpy as np

import emu_py

_HERE = os.path.dirname(os.path.abspath(__file__))
a1mpc = emu_py.a1mpc
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "ext_warm.mk", "liba1mpc_emu_ext_warm.so"])
        _LIB = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_ext_warm.so"))
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _solve(fn, cfg, st, sched, normals, warm, shift, order, nthreads, want_u):
    B = st["contact"].shape[0]
    assert warm.dtype == np.uint32 and warm.shape == (B, 4 + 4 * cfg.horizon) and warm.flags["C_CONTIGUOUS"]
    arrs = [np.ascontiguousarray(st[k], dtype=np.float64) for k in ("x0", "rot", "foot", "ref")]
    contact = np.ascontiguousarray(st["contact"], dtype=np.uint32)
    inp = a1mpc.Inputs(_p(arrs[0]), _p(arrs[1]), _p(arrs[2]), _p(arrs[3]), _p(contact), B)
    f = np.zeros((12, B)); status = np.full(B, -7, dtype=np.int32); iters = np.zeros(B, dtype=np.int32)
    u = np.zeros((12 * cfg.horizon, B)) if want_u else None
    out = a1mpc.Outputs(_p(f), _p(status), _p(iters), _p(u), B)
    sc = np.ascontiguousarray(sched, dtype=np.uint32) if sched is not None else None
    nm = np.ascontiguousarray(normals, dtype=np.float64) if normals is not None else None
    rc = fn(C.byref(cfg), B, C.byref(inp), _p(sc), _p(nm), C.byref(out), order, nthreads, _p(warm), shift)
    assert rc == 0, rc
    return (f, status, iters, u) if want_u else (f, status, iters)


def solve(cfg, st, sched, normals, warm, shift=1, order=0, nthreads=8, want_u=False):
    """a1mpc_solve_batch_ext_warm on the general four-leg kernel; warm [B, 4 + 4N] u32 is updated in place"""
    return _solve(lib().emu_solve_ext_warm, cfg, st, sched, normals, warm, shift, order, nthreads, want_u)


def solve_sched2(cfg, st, sched, normals, warm, shift=1, order=0, nthreads=8, want_u=False):
    """the same on the compacted two-feet kernel (every step of every schedule must have exactly two stance feet)"""
    return _solve(lib().emu_solve_sched2_warm, cfg, st, sched, normals, warm, shift, order, nthreads, want_u)
