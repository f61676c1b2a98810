"""ctypes binding of oracle/liba1mpc_command_oracle.so (command_oracle.cpp, built by `make -C oracle -f command.mk`): the oracle of
a1mpc_orientation_batch / a1mpc_command_batch.  TEST INFRASTRUCTURE; the product (a1-qp-mpc-controller_b200/) never imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liba1mpc_command_oracle.so")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "command_oracle.cpp")):
            subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "command.mk", "liba1mpc_command_oracle.so"])
        L = C.CDLL(_SO)
        L.oracle_quat_to_euler.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        L.oracle_window.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.oracle_imu_new.restype = C.c_void_p
        L.oracle_imu_new.argtypes = [C.c_int, C.c_int]
        L.oracle_imu_free.argtypes = [C.c_void_p]
        L.oracle_orientation.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 9
        L.oracle_command_new.restype = C.c_void_p
        L.oracle_command_new.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.oracle_command_free.argtypes = [C.c_void_p]
        L.oracle_command.argtypes = [C.c_void_p, C.c_int, C.c_double] + [C.c_void_p] * 7
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _a(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def quat_to_euler(quat):
    """quat [4,n] (w, x, y, z) -> euler [3,n]"""
    q = _a(quat)
    e = np.zeros((3, q.shape[1]))
    assert lib().oracle_quat_to_euler(q.shape[1], _p(q), _p(e)) == 0
    return e


def window(W, x):
    """one MovingWindowFilter(W) over the samples x [T] -> the T averages"""
    x = _a(x)
    y = np.zeros_like(x)
    assert lib().oracle_window(int(W), x.shape[0], _p(x), _p(y)) == 0
    return y


class Orientation:
    """the orientation stage for B robots; the six IMU filters per robot (filtered=True) stay inside the object"""

    def __init__(self, B, filtered=True):
        self.L, self.B = lib(), int(B)
        self.h = C.c_void_p(self.L.oracle_imu_new(self.B, int(bool(filtered))))

    def __call__(self, quat, gyro, acc=None):
        """-> dict rot, rot_z [9,B], euler, ang_vel, imu_acc (None without acc), imu_ang_vel [3,B]"""
        B = self.B
        q, g = _a(quat), _a(gyro)
        a = _a(acc) if acc is not None else None
        o = dict(rot=np.zeros((9, B)), rot_z=np.zeros((9, B)), euler=np.zeros((3, B)), ang_vel=np.zeros((3, B)),
                 imu_acc=np.zeros((3, B)) if a is not None else None, imu_ang_vel=np.zeros((3, B)))
        assert self.L.oracle_orientation(self.h, B, _p(q), _p(g), _p(a), *[_p(o[k]) for k in ("rot", "rot_z", "euler", "ang_vel", "imu_acc",
                                                                                             "imu_ang_vel")]) == 0
        return o

    def __del__(self):
        try:
            self.L.oracle_imu_free(self.h)
        except Exception:
            pass


class Command:
    """main_update's front half for B robots with the adapter's state inside the object.  variant 0 Gazebo, 1 hardware, 2 Isaac."""

    def __init__(self, B, variant=0, body_height=0.3, hmin=0.1, hmax=0.32, kp_linear=(120.0, 120.0, 500.0), lock=(120.0, 120.0)):
        self.L, self.B = lib(), int(B)
        kp, lk = _a(kp_linear), _a(lock)
        self.h = C.c_void_p(self.L.oracle_command_new(self.B, int(variant), body_height, hmin, hmax, _p(kp), _p(lk)))

    def __call__(self, dt, cmd, root_pos, euler_d1=None):
        """cmd [7,B], root_pos [3,B]; euler_d1 [B] = root_euler_d[1] as compute_grf left it (None: the object's own) ->
        movement_mode [B], kp_linear [3,B], ref [9,B], des [12,B]"""
        B = self.B
        c, pos = _a(cmd), _a(root_pos)
        e1 = _a(euler_d1) if euler_d1 is not None else None
        mode = np.zeros(B, dtype=np.uint32); kp = np.zeros((3, B)); ref = np.zeros((9, B)); des = np.zeros((12, B))
        assert self.L.oracle_command(self.h, B, C.c_double(dt), _p(c), _p(pos), _p(e1), _p(mode), _p(kp), _p(ref), _p(des)) == 0
        return mode, kp, ref, des

    def __del__(self):
        try:
            self.L.oracle_command_free(self.h)
        except Exception:
            pass
