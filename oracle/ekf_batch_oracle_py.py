"""ctypes binding of oracle/liba1mpc_ekf_batch_oracle.so (ekf_batch_oracle.cpp, built by `make -C oracle -f ekf_batch.mk`): the
oracle's A1BasicEKF update (oracle_py.ekf_update) for a batch of robots on host threads, in the layout of a1mpc_ekf_update_batch.
TEST INFRASTRUCTURE; the product (a1-qp-mpc-controller_b200/) never imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liba1mpc_ekf_batch_oracle.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "ekf_batch_oracle.cpp")):
            subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "ekf_batch.mk", "liba1mpc_ekf_batch_oracle.so"])
        L = C.CDLL(_SO)
        L.oracle_ekf_update_batch.argtypes = [C.c_int, C.c_double, C.c_int] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 5
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def ekf_update_batch(state, dt, assume_flat_ground, movement_mode, imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel, foot_force, nthreads=1):
    """oracle_py.ekf_update for B robots, in place on state [B,342] (x[18], P[18,18] per robot); inputs [rows,B].  Returns root_pos
    [3,B], root_lin_vel [3,B], estimated_contacts [B], rc [B].  A robot with rc != 0 keeps its state, and its outputs are NaN (root_pos,
    root_lin_vel) and 0xffffffff (estimated_contacts)."""
    B = state.shape[0]
    assert state.shape == (B, 342) and state.dtype == np.float64 and state.flags["C_CONTIGUOUS"]
    mm = np.ascontiguousarray(movement_mode, dtype=np.uint32)
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel, foot_force)]
    assert mm.shape == (B,) and [v.shape for v in a] == [(3, B), (3, B), (9, B), (12, B), (12, B), (4, B)]
    pos = np.full((3, B), np.nan); vel = np.full((3, B), np.nan); ec = np.full(B, 0xffffffff, dtype=np.uint32); rc = np.full(B, -1, dtype=np.int32)
    lib().oracle_ekf_update_batch(B, dt, int(assume_flat_ground), _ptr(mm), *[_ptr(v) for v in a], int(nthreads), _ptr(state),
                                  _ptr(pos), _ptr(vel), _ptr(ec), _ptr(rc))
    return pos, vel, ec, rc
