"""ctypes binding of the CPU block emulator of the multi-rate tick's kernels (tests/emu/liba1mpc_emu_tick_rate.so, built from
emu_tick_rate.cpp by tick_rate.mk).  TEST INFRASTRUCTURE, the companion of emu_tick_reset_py.py.  Every array is a contiguous float64 /
uint32 / int32 / uint8 numpy array, dense [rows][B] (the warm slots [B][WARM_HDR + 4N]), updated in place."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "tick_rate.mk", "all"])
        L = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_tick_rate.so"))
        L.emu_rate_sizes.argtypes = [C.c_void_p]
        L.emu_rate_pack.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 6
        L.emu_tick_rate.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5
        L.emu_tick_rate_reset.argtypes = [C.c_int] + [C.c_void_p] * 3
        L.emu_plan_forces.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    assert a.flags.c_contiguous and a.dtype in (np.float64, np.uint32, np.int32, np.uint8), a.dtype
    return a.ctypes.data_as(C.c_void_p)


def sizes():
    """dict of rec (REC_DOUBLES), rec_ext (REC_EXT_DOUBLES) and warm_hdr (WARM_HDR)"""
    out = np.zeros(3, dtype=np.int32)
    lib().emu_rate_sizes(out.ctypes.data_as(C.c_void_p))
    return dict(zip(("rec", "rec_ext", "warm_hdr"), (int(v) for v in out)))


def pack(kind, horizon, st, sched, normals, runs, period, rec, cap, count, out, warm):
    """kind 0 pack_kernel, 1 (warm_forget_no_contact_kernel +) pack_ext_kernel, 2 the same with pack_ext2_kernel; runs not None: their
    masked variants.  st: x0, rot, foot, ref, contact; out: f_body, status, iters, u_full (None allowed); rec, count, out, warm in place"""
    B = st["contact"].shape[0]
    assert lib().emu_rate_pack(kind, B, horizon, *(_p(st[k]) for k in ("x0", "rot", "foot", "ref", "contact")), _p(sched), _p(normals), _p(runs),
                               period, _p(rec), cap, _p(count), *(_p(out.get(k)) for k in ("f_body", "status", "iters", "u_full")), _p(warm)) == 0


def tick_rate(B, period, horizon, runs, since, rot, plan, f_body):
    assert lib().emu_tick_rate(B, period, horizon, _p(runs), _p(since), _p(rot), _p(plan), _p(f_body)) == 0


def tick_rate_reset(B, mask, runs, since):
    assert lib().emu_tick_rate_reset(B, _p(mask), _p(runs), _p(since)) == 0


def plan_forces(B, horizon, rot, u_full, step, f_body):
    assert lib().emu_plan_forces(B, horizon, _p(rot), _p(u_full), _p(step), _p(f_body)) == 0
