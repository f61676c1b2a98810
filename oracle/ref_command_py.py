"""ctypes binding of oracle/_ref/libref_command.so: the REFERENCE'S OWN Utils::quat_to_euler (utils/Utils.cpp compiled unmodified against
the header stand-ins of oracle/ref_shim/) and its MovingWindowFilter (utils/filter.hpp), through ref_command_wrap.cpp
(`make -C oracle -f command.mk ref`).  TEST INFRASTRUCTURE.

Exists only where the reference sources were present when that build ran.  No GPU test may depend on it: tests use
tests/golden/command_v1.npz (tests/golden/make_command_golden.py) and call `available()` before touching anything here."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libref_command.so")
_LIB = None


def available():
    return os.path.exists(_SO)


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(_SO)
        L.ref_quat_to_euler.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        L.ref_window.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def quat_to_euler(quat):
    """Utils::quat_to_euler(Quaterniond(w, x, y, z)) column by column: quat [4,n] -> euler [3,n]"""
    q = np.ascontiguousarray(quat, dtype=np.float64)
    e = np.zeros((3, q.shape[1]))
    assert lib().ref_quat_to_euler(q.shape[1], _p(q), _p(e)) == 0
    return e


def window(W, x):
    """MovingWindowFilter(W).CalculateAverage over the samples x [T] -> the T averages"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.zeros_like(x)
    assert lib().ref_window(int(W), x.shape[0], _p(x), _p(y)) == 0
    return y
