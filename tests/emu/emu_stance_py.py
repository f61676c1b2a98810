"""ctypes binding of the CPU block emulator of a1mpc_stance_qp_batch (tests/emu/liba1mpc_emu_stance.so, built from emu_stance.cpp by
stance.mk).  TEST INFRASTRUCTURE, the companion of emu_py.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "stance.mk", "liba1mpc_emu_stance.so"])
        _LIB = C.CDLL(os.path.join(_HERE, "liba1mpc_emu_stance.so"))
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def stance_qp(x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, mass, want_acc=True, order=0):
    """a1mpc_stance_qp_batch on the emulator, batch-major host arrays (ld = B) -> f_body [12,B], status [B] (, root_acc [6,B])"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x0, rot, rot_z, foot)]
    contact = np.ascontiguousarray(contact, dtype=np.uint32)
    d, kpl = np.ascontiguousarray(des, dtype=np.float64), np.ascontiguousarray(kp_linear, dtype=np.float64)
    gains = np.ascontiguousarray(np.concatenate([kd_linear, kp_angular, kd_angular]), dtype=np.float64)
    B = contact.shape[0]
    f = np.full((12, B), np.nan); status = np.full(B, -7, dtype=np.int32)
    acc = np.full((6, B), np.nan) if want_acc else None
    assert lib().emu_stance_qp(B, C.c_size_t(B), *[_p(v) for v in a], _p(contact), _p(d), _p(kpl), _p(gains), C.c_double(mass), _p(f), _p(status),
                               _p(acc), int(order)) == 0
    return (f, status, acc) if want_acc else (f, status)
