"""ctypes binding of liba1mpc.so (the C ABI in include/a1mpc.h).

This file is glue for tests/ and bench.py: it marshals numpy arrays to the C entry points and nothing
else.  There is no Python compute path and no fallback: if the shared library is missing or no H100 is
visible, construction fails loudly.  C++ hosts use include/a1mpc.h (or the ConvexMpcBatch /
A1RobotControlBatch shims under host/) directly.
"""
import ctypes as C
import os
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("A1MPC_LIB", os.path.join(_HERE, "liba1mpc.so"))   # A1MPC_LIB: developer A/B builds only

STATUS_OPTIMAL, STATUS_IPM_ONLY, STATUS_MAXITER, STATUS_NUMERICAL, STATUS_NO_CONTACT = 0, 1, 2, 3, 4

EXPORTS = [
    "a1mpc_default_config", "a1mpc_create", "a1mpc_destroy", "a1mpc_last_error", "a1mpc_device_count",
    "a1mpc_solve_batch", "a1mpc_warm_bytes", "a1mpc_warm_reset", "a1mpc_solve_batch_warm", "a1mpc_solve_batch_ext", "a1mpc_solve_batch_ext_warm", "a1mpc_build_qp_batch", "a1mpc_qp_mats_batch", "a1mpc_solve_dense_batch",
    "a1mpc_grf_qp_batch", "a1mpc_stance_qp_batch", "a1mpc_stance_qp_batch_ext", "a1mpc_joint_torques_batch", "a1mpc_leg_kinematics_batch", "a1mpc_ekf_bytes", "a1mpc_ekf_init_batch", "a1mpc_ekf_update_batch", "a1mpc_update_plan_batch",
    "a1mpc_swing_bytes", "a1mpc_swing_init_batch", "a1mpc_swing_legs_batch", "a1mpc_terrain_pitch_batch", "a1mpc_terrain_normals_batch", "a1mpc_surface_normals_batch",
    "a1mpc_imu_bytes", "a1mpc_imu_init_batch", "a1mpc_orientation_batch", "a1mpc_command_bytes", "a1mpc_command_init_batch", "a1mpc_command_batch",
    "a1mpc_default_tick_params", "a1mpc_tick_create", "a1mpc_tick_reset", "a1mpc_tick_reset_robots", "a1mpc_tick_set_terrain", "a1mpc_tick_set_stance_terrain", "a1mpc_tick_set_mpc_period", "a1mpc_tick_set_gaits", "a1mpc_gait_row", "a1mpc_update_plan_gait_batch", "a1mpc_swing_legs_gait_batch", "a1mpc_plan_forces_batch", "a1mpc_tick_run", "a1mpc_tick_destroy",
    "a1mpc_device_alloc", "a1mpc_device_free", "a1mpc_host_alloc", "a1mpc_host_free",
    "a1mpc_memcpy_h2d", "a1mpc_memcpy_d2h", "a1mpc_sync", "a1mpc_event_create", "a1mpc_event_destroy",
    "a1mpc_event_record", "a1mpc_event_elapsed_ms", "a1mpc_launch_count", "a1mpc_measure_fp64_peak",
    "a1mpc_flush_l2", "a1mpc_profile_begin", "a1mpc_profile_end", "a1mpc_nccl_unique_id", "a1mpc_nccl_init", "a1mpc_allgather_forces",
    "a1mpc_qp_rollout_batch", "a1mpc_peer_gather_create", "a1mpc_peer_gather_connect", "a1mpc_peer_gather_buffer", "a1mpc_peer_gather_wait", "a1mpc_peer_gather_status", "a1mpc_peer_gather_destroy", "a1mpc_gen_states", "a1mpc_gen_schedule",
]


class Config(C.Structure):
    _fields_ = [("horizon", C.c_int), ("precision", C.c_int), ("dt", C.c_double),
                ("mu", C.c_double), ("fz_min", C.c_double), ("fz_max", C.c_double),
                ("mass", C.c_double), ("inertia", C.c_double * 9),
                ("q", C.c_double * 13), ("r", C.c_double * 12),
                ("max_iter", C.c_int), ("tol", C.c_double)]


class Inputs(C.Structure):
    _fields_ = [("x0", C.c_void_p), ("rot", C.c_void_p), ("foot", C.c_void_p), ("ref", C.c_void_p),
                ("contact", C.c_void_p), ("ld", C.c_size_t)]


class GaitParams(C.Structure):
    _fields_ = [("counter_per_gait", C.c_double), ("counter_per_swing", C.c_double), ("control_dt", C.c_double),
                ("default_foot_pos", C.c_double * 12), ("foot_delta_x_limit", C.c_double), ("foot_delta_y_limit", C.c_double),
                ("horizon", C.c_int)]


def default_gait_params(horizon=10):
    """A1CtrlStates.h:23-24, 45-47, 332; A1Params.h:44-45"""
    g = GaitParams()
    g.counter_per_gait, g.counter_per_swing, g.control_dt = 240.0, 120.0, 0.0025
    g.default_foot_pos[:] = [0.17, 0.17, -0.17, -0.17, 0.15, -0.15, 0.15, -0.15, -0.35, -0.35, -0.35, -0.35]
    g.foot_delta_x_limit, g.foot_delta_y_limit, g.horizon = 0.1, 0.1, horizon
    return g


VARIANT_GAZEBO, VARIANT_HARDWARE, VARIANT_ISAAC = 0, 1, 2


class CommandParams(C.Structure):
    _fields_ = [("variant", C.c_int), ("body_height", C.c_double), ("body_height_min", C.c_double), ("body_height_max", C.c_double),
                ("kp_linear", C.c_double * 3), ("kp_linear_lock", C.c_double * 2)]


def default_command_params(variant=VARIANT_GAZEBO):
    """the adapter's initial joy_cmd_body_height (GazeboA1ROS.h:130, HardwareA1ROS.h:107, IsaacA1ROS.h:80), JOY_CMD_BODY_HEIGHT_MIN / _MAX
    (A1Params.h:16-17) and the ROS-parameter defaults of kp_linear and its lock gains (A1CtrlStates.h:270-301)"""
    c = CommandParams()
    c.variant = variant
    c.body_height = {VARIANT_GAZEBO: 0.3, VARIANT_HARDWARE: 0.12, VARIANT_ISAAC: 0.32}.get(variant, 0.3)
    c.body_height_min, c.body_height_max = 0.1, 0.32
    c.kp_linear[:] = [120.0, 120.0, 500.0]
    c.kp_linear_lock[:] = [120.0, 120.0]
    return c


TICK_QP, TICK_MPC = 0, 1
TERRAIN_FLAT, TERRAIN_ESTIMATED, TERRAIN_GIVEN = 0, 1, 2   # a1mpc_tick_set_terrain
PLAYBACK_HOLD, PLAYBACK_PLAN = 0, 1                        # a1mpc_tick_set_mpc_period
GAIT_TROT, GAIT_PACE, GAIT_BOUND, GAIT_PRONK, GAIT_WALK = 1, 2, 3, 4, 5   # a1mpc_gait_row


class TickParams(C.Structure):
    _fields_ = [("mode", C.c_int), ("use_terrain_adapt", C.c_int), ("assume_flat_ground", C.c_int), ("gait", GaitParams), ("command", CommandParams),
                ("rho_opt", C.c_double * 12), ("rho_fix", C.c_double * 20), ("kp_foot", C.c_double * 12), ("kd_foot", C.c_double * 12),
                ("km_foot", C.c_double * 3), ("torques_gravity", C.c_double * 12), ("kd_linear", C.c_double * 3), ("kp_angular", C.c_double * 3),
                ("kd_angular", C.c_double * 3)]


TICK_INPUTS = ("quat", "gyro", "acc", "joint_pos", "joint_vel", "foot_force", "cmd", "gait_counter_speed")
TICK_OUTPUTS = ("tau", "f_body", "status", "contacts", "movement_mode", "x0", "ref")


class TickInputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in TICK_INPUTS]


class TickOutputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in TICK_OUTPUTS]


def default_tick_params(variant=VARIANT_GAZEBO, mode=TICK_MPC):
    """a1mpc_default_tick_params: the reference's launch parameters of one adapter and stance_leg_control_type"""
    tp = TickParams()
    _check(lib().a1mpc_default_tick_params(variant, mode, C.byref(tp)))
    return tp


class InputsExt(C.Structure):
    _fields_ = [("contact_sched", C.c_void_p), ("normals", C.c_void_p)]


class Outputs(C.Structure):
    _fields_ = [("f_body", C.c_void_p), ("status", C.c_void_p), ("iters", C.c_void_p), ("u_full", C.c_void_p),
                ("ld", C.c_size_t)]


_lib = None


def lib():
    """loads liba1mpc.so; raises if it has not been built (python __graft_entry__.py build / make)"""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("liba1mpc.so is missing: run `make` (or __graft_entry__.build()) first; "
                               "there is no Python/CPU fallback for the engine")
        l = C.CDLL(LIB_PATH)
        l.a1mpc_last_error.restype = C.c_char_p
        l.a1mpc_launch_count.restype = C.c_int64
        l.a1mpc_warm_bytes.restype = C.c_size_t
        l.a1mpc_ekf_bytes.restype = C.c_size_t
        l.a1mpc_launch_count.argtypes = [C.c_void_p]
        for name in ("a1mpc_device_alloc", "a1mpc_host_alloc"):
            getattr(l, name).argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
        for name in ("a1mpc_device_free", "a1mpc_host_free", "a1mpc_event_destroy", "a1mpc_event_record"):
            getattr(l, name).argtypes = [C.c_void_p, C.c_void_p]
        for name in ("a1mpc_memcpy_h2d", "a1mpc_memcpy_d2h"):
            getattr(l, name).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        l.a1mpc_sync.argtypes = [C.c_void_p]
        l.a1mpc_flush_l2.argtypes = [C.c_void_p]
        l.a1mpc_peer_gather_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        l.a1mpc_peer_gather_connect.argtypes = [C.c_void_p, C.c_char_p]
        l.a1mpc_peer_gather_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        l.a1mpc_peer_gather_wait.argtypes = [C.c_void_p]
        l.a1mpc_peer_gather_status.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        l.a1mpc_peer_gather_destroy.argtypes = [C.c_void_p]
        l.a1mpc_destroy.argtypes = [C.c_void_p]
        l.a1mpc_event_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        l.a1mpc_event_elapsed_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
        l.a1mpc_solve_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(Inputs), C.POINTER(Outputs)]
        l.a1mpc_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(Config), C.c_int]
        l.a1mpc_default_config.argtypes = [C.POINTER(Config)]
        l.a1mpc_warm_bytes.argtypes = [C.c_void_p, C.c_int]
        l.a1mpc_warm_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.a1mpc_solve_batch_warm.argtypes = [C.c_void_p, C.c_int, C.POINTER(Inputs), C.POINTER(Outputs), C.c_void_p, C.c_int]
        l.a1mpc_leg_kinematics_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 10
        l.a1mpc_ekf_bytes.argtypes = [C.c_int]
        l.a1mpc_ekf_init_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        l.a1mpc_ekf_update_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_int] + [C.c_void_p] * 11
        l.a1mpc_solve_batch_ext.argtypes = [C.c_void_p, C.c_int, C.POINTER(Inputs), C.POINTER(InputsExt), C.POINTER(Outputs)]
        l.a1mpc_solve_batch_ext_warm.argtypes = [C.c_void_p, C.c_int, C.POINTER(Inputs), C.POINTER(InputsExt), C.POINTER(Outputs), C.c_void_p, C.c_int]
        l.a1mpc_gen_schedule.argtypes = [C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        l.a1mpc_build_qp_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(Inputs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        l.a1mpc_qp_mats_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 6
        l.a1mpc_qp_rollout_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 8
        l.a1mpc_solve_dense_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        l.a1mpc_grf_qp_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
        l.a1mpc_stance_qp_batch.argtypes = [C.c_void_p, C.c_int, C.c_size_t] + [C.c_void_p] * 13
        l.a1mpc_stance_qp_batch_ext.argtypes = [C.c_void_p, C.c_int, C.c_size_t] + [C.c_void_p] * 14
        l.a1mpc_joint_torques_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
        l.a1mpc_update_plan_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(GaitParams)] + [C.c_void_p] * 13
        l.a1mpc_swing_bytes.restype = C.c_size_t
        l.a1mpc_swing_bytes.argtypes = [C.c_int]
        l.a1mpc_swing_init_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.a1mpc_swing_legs_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(GaitParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_double] + [C.c_void_p] * 10
        l.a1mpc_terrain_pitch_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        l.a1mpc_terrain_normals_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                  C.c_void_p]
        l.a1mpc_surface_normals_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        for name in ("a1mpc_imu_bytes", "a1mpc_command_bytes"):
            getattr(l, name).restype = C.c_size_t
            getattr(l, name).argtypes = [C.c_int]
        l.a1mpc_imu_init_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.a1mpc_orientation_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7 + [C.c_size_t, C.c_void_p, C.c_void_p]
        l.a1mpc_command_init_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(CommandParams), C.c_void_p, C.c_size_t]
        l.a1mpc_command_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        l.a1mpc_default_tick_params.argtypes = [C.c_int, C.c_int, C.POINTER(TickParams)]
        l.a1mpc_tick_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(TickParams), C.POINTER(C.c_void_p)]
        l.a1mpc_tick_reset.argtypes = [C.c_void_p]
        l.a1mpc_tick_reset_robots.argtypes = [C.c_void_p, C.c_void_p]
        l.a1mpc_tick_set_terrain.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.a1mpc_tick_set_stance_terrain.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.a1mpc_tick_set_mpc_period.argtypes = [C.c_void_p, C.c_int, C.c_int]
        l.a1mpc_tick_set_gaits.argtypes = [C.c_void_p, C.c_void_p]
        l.a1mpc_gait_row.argtypes = [C.c_int, C.c_void_p]
        l.a1mpc_update_plan_gait_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(GaitParams)] + [C.c_void_p] * 14
        l.a1mpc_swing_legs_gait_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(GaitParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_double] + [C.c_void_p] * 10
        l.a1mpc_plan_forces_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4
        l.a1mpc_tick_run.argtypes = [C.c_void_p, C.c_double, C.POINTER(TickInputs), C.POINTER(TickOutputs)]
        l.a1mpc_tick_destroy.argtypes = [C.c_void_p]
        l.a1mpc_gen_states.argtypes = [C.c_int, C.c_uint64, C.c_int] + [C.c_void_p] * 5
        l.a1mpc_measure_fp64_peak.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        l.a1mpc_profile_begin.argtypes = [C.c_void_p, C.c_int]
        l.a1mpc_profile_end.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        l.a1mpc_nccl_unique_id.argtypes = [C.c_void_p]
        l.a1mpc_nccl_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.a1mpc_allgather_forces.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        _lib = l
    return _lib


class A1MpcError(RuntimeError):
    pass


def _check(rc):
    if rc != 0:
        raise A1MpcError("a1mpc error %d: %s" % (rc, (lib().a1mpc_last_error() or b"").decode()))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def default_config(**kw):
    c = Config()
    lib().a1mpc_default_config(C.byref(c))
    for k, v in kw.items():
        if k in ("inertia", "q", "r"):
            getattr(c, k)[:] = v
        else:
            setattr(c, k, v)
    return c


def gen_states(B, config_id=2, stream=0):
    """deterministic synthetic trot-gait batch (SURVEY 8d) -> dict of host SoA arrays"""
    x0 = np.zeros((12, B)); rot = np.zeros((9, B)); foot = np.zeros((12, B)); ref = np.zeros((9, B))
    contact = np.zeros(B, dtype=np.uint32)
    rc = lib().a1mpc_gen_states(config_id, stream, B, _p(x0), _p(rot), _p(foot), _p(ref), _p(contact))
    _check(rc)
    return dict(x0=x0, rot=rot, foot=foot, ref=ref, contact=contact)


def gen_schedule(B, horizon, config_id=4, stream=0):
    """config-4 extras: per-step contact schedule [N,B] and per-foot terrain normals [12,B]"""
    sched = np.zeros((horizon, B), dtype=np.uint32); normals = np.zeros((12, B))
    _check(lib().a1mpc_gen_schedule(config_id, stream, B, horizon, _p(sched), _p(normals)))
    return sched, normals


class DeviceBatch:
    """device-resident SoA inputs + outputs of one batch (ld = B)"""

    def __init__(self, eng, B, want_u=False, want_iters=True):
        self.eng, self.B = eng, B
        N = eng.cfg.horizon
        es = np.dtype(eng.ftype).itemsize
        self.x0 = eng.dalloc(12 * B * es); self.rot = eng.dalloc(9 * B * es); self.foot = eng.dalloc(12 * B * es)
        self.ref = eng.dalloc(9 * B * es); self.contact = eng.dalloc(B * 4)
        self.f_body = eng.dalloc(12 * B * es); self.status = eng.dalloc(B * 4)
        self.iters = eng.dalloc(B * 4) if want_iters else None
        self.u_full = eng.dalloc(12 * N * B * es) if want_u else None
        self.inp = Inputs(self.x0, self.rot, self.foot, self.ref, self.contact, B)
        self.out = Outputs(self.f_body, self.status, self.iters, self.u_full, B)

    def upload(self, st):
        e = self.eng
        for name in ("x0", "rot", "foot", "ref", "contact"):
            a = np.ascontiguousarray(st[name], dtype=(np.uint32 if name == "contact" else e.ftype))
            _check(lib().a1mpc_memcpy_h2d(e.h, getattr(self, name), _p(a), a.nbytes))
        e.sync()

    def download(self):
        e, B = self.eng, self.B
        f = np.zeros((12, B), dtype=e.ftype); status = np.zeros(B, dtype=np.int32)
        _check(lib().a1mpc_memcpy_d2h(e.h, _p(f), self.f_body, f.nbytes))
        _check(lib().a1mpc_memcpy_d2h(e.h, _p(status), self.status, status.nbytes))
        e.sync()
        return f, status

    def free(self):
        for name in ("x0", "rot", "foot", "ref", "contact", "f_body", "status", "iters", "u_full"):
            p = getattr(self, name)
            if p:
                lib().a1mpc_device_free(self.eng.h, p)
                setattr(self, name, None)


def gait_row(gait_type):
    """a1mpc_gait_row: one robot's gait row [6] (offsets FL FR RL RR, counter_per_gait, counter_per_swing) of GAIT_TROT / _PACE / _BOUND /
    _PRONK / _WALK; np.repeat(gait_row(t)[:, None], B, axis=1) makes the [6][B] rows of Tick.set_gaits"""
    row = np.zeros(6)
    _check(lib().a1mpc_gait_row(int(gait_type), _p(row)))
    return row


class Tick:
    """a whole control tick for B robots (a1mpc_tick_*): owns the controller state; raw sensor arrays in, joint torques out.

    In MPC mode params.gait.horizon picks how the solve is posed: 0 (the default) holds the current contact pattern over the horizon as
    the reference does; the engine's horizon runs the scheduled tick, whose solve sees the gait's planned contacts over the horizon (step 0
    the swing stage's contacts) and does not take part in the fused collect.  Any other value is rejected; QP mode ignores it.
    set_terrain picks where the MPC solve's friction pyramids stand: world z (the default), the estimated walking surface or the caller's
    normals; set_stance_terrain does the same for the QP-mode stance QP.  set_mpc_period runs the MPC solve of each robot on every k-th
    run only, staggered across the batch."""

    _SHAPES = dict(quat=(4,), gyro=(3,), acc=(3,), joint_pos=(12,), joint_vel=(12,), foot_force=(4,), cmd=(7,), gait_counter_speed=(4,))

    def __init__(self, eng, B, params=None):
        self.eng, self.B = eng, B
        self.params = params if params is not None else default_tick_params()
        t = C.c_void_p()
        _check(lib().a1mpc_tick_create(eng.h, B, C.byref(self.params), C.byref(t)))
        self.t = t
        eng._ticks.add(self)   # Engine.close destroys its ticks first: a tick must go before its handle

    def run(self, dt, quat, gyro, acc, joint_pos, joint_vel, foot_force, cmd, gait_counter_speed):
        """one tick on host arrays ([rows][B] float64) -> (tau [12][B], dict of f_body, status, contacts, movement_mode, x0 and, in MPC
        mode, ref)"""
        B = self.B
        args = dict(quat=quat, gyro=gyro, acc=acc, joint_pos=joint_pos, joint_vel=joint_vel, foot_force=foot_force, cmd=cmd,
                    gait_counter_speed=gait_counter_speed)
        arrs = {}
        for k, a in args.items():
            arrs[k] = np.ascontiguousarray(a, dtype=np.float64)
            if arrs[k].shape != self._SHAPES[k] + (B,):
                raise ValueError("%s must have shape %s" % (k, self._SHAPES[k] + (B,)))
        outs = dict(tau=np.zeros((12, B)), f_body=np.zeros((12, B)), status=np.zeros(B, dtype=np.int32), contacts=np.zeros(B, dtype=np.uint32),
                    movement_mode=np.zeros(B, dtype=np.uint32), x0=np.zeros((12, B)))
        if self.params.mode == TICK_MPC:
            outs["ref"] = np.zeros((9, B))
        self.run_ptrs(dt, TickInputs(*[arrs[k].ctypes.data for k in TICK_INPUTS]),
                      TickOutputs(*[outs[k].ctypes.data if k in outs else None for k in TICK_OUTPUTS]))
        tau = outs.pop("tau")
        return tau, outs

    def run_ptrs(self, dt, inputs, outputs):
        """one tick on a TickInputs / TickOutputs of device pointers (asynchronous on the handle's stream) or host pointers"""
        _check(lib().a1mpc_tick_run(self.t, dt, C.byref(inputs), C.byref(outputs)))

    def reset(self):
        _check(lib().a1mpc_tick_reset(self.t))

    def reset_robots(self, mask):
        """a1mpc_tick_reset_robots on a host mask: numpy bool or uint8 [B]; robot b with mask[b] != 0 starts over as after reset(), the
        others keep their state.  Copies the mask and synchronises; reset_robots_ptr takes a device mask without either"""
        m = np.asarray(mask)
        if m.dtype not in (np.bool_, np.uint8) or m.shape != (self.B,):
            raise ValueError("mask must be a bool or uint8 array of shape (%d,)" % self.B)
        m = np.ascontiguousarray(m).view(np.uint8)
        self.reset_robots_ptr(m.ctypes.data)

    def reset_robots_ptr(self, ptr):
        """a1mpc_tick_reset_robots on a pointer to B uint8 / bool, e.g. a torch bool tensor's data_ptr(): device memory only enqueues work on
        the handle's stream, host memory is copied and synchronised"""
        _check(lib().a1mpc_tick_reset_robots(self.t, ptr))

    def set_terrain(self, source, normals_ptr=0):
        """a1mpc_tick_set_terrain: TERRAIN_FLAT (world-z pyramids, the default), TERRAIN_ESTIMATED (the terrain stage's fitted surface
        normal) or TERRAIN_GIVEN with normals_ptr a device pointer to [12][B] float64 per-foot normals, e.g. a torch tensor's data_ptr(),
        read by every later run.  MPC mode only for the non-flat sources"""
        _check(lib().a1mpc_tick_set_terrain(self.t, int(source), normals_ptr or None))

    def set_stance_terrain(self, source, normals_ptr=0):
        """a1mpc_tick_set_stance_terrain, the QP-mode counterpart of set_terrain: TERRAIN_FLAT (world-z pyramids, the default),
        TERRAIN_ESTIMATED (the walking surface fitted through the recent-contact points) or TERRAIN_GIVEN with normals_ptr a device pointer to
        [12][B] float64 per-foot normals, read by every later run.  QP mode only"""
        _check(lib().a1mpc_tick_set_stance_terrain(self.t, int(source), normals_ptr or None))

    def set_mpc_period(self, period, playback=PLAYBACK_PLAN):
        """a1mpc_tick_set_mpc_period: robot b solves the MPC on its runs n with n == 0 or n % period == b % period (period 1..N, MPC mode);
        on its other runs PLAYBACK_PLAN applies the step of its last solve's plan that belongs to the run, rotated by this run's rot, and
        PLAYBACK_HOLD keeps the forces and status of its last solve.  Every robot solves on the next run"""
        _check(lib().a1mpc_tick_set_mpc_period(self.t, int(period), int(playback)))

    def set_gaits(self, rows):
        """a1mpc_tick_set_gaits on host rows: float64 [6][B] (rows 0-3 the standstill counters FL FR RL RR, row 4 counter_per_gait, row 5
        counter_per_swing; gait_row builds one column), or None for the reference's trot.  The rows are checked (a bad one raises A1MpcError
        naming the robot and leaves the previous gaits in force); cps and cpg apply from the next run, the offsets when a robot stands"""
        if rows is None:
            self.set_gaits_ptr(0)
            return
        g = np.ascontiguousarray(rows, dtype=np.float64)
        if g.shape != (6, self.B):
            raise ValueError("gait rows must have shape (6, %d)" % self.B)
        self.set_gaits_ptr(g.ctypes.data)

    def set_gaits_ptr(self, ptr):
        """a1mpc_tick_set_gaits on a pointer to [6][B] float64, e.g. a torch device tensor's data_ptr(); 0 returns to the trot"""
        _check(lib().a1mpc_tick_set_gaits(self.t, ptr or None))

    def close(self):
        """a1mpc_tick_destroy; a tick whose Engine is closed has already been destroyed by Engine.close"""
        if self.t and self.eng.h:
            lib().a1mpc_tick_destroy(self.t)
        self.t = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """one handle = one H100 + one stream (a1mpc_create / a1mpc_destroy)"""

    def __init__(self, cfg=None, device=0):
        self.cfg = cfg if cfg is not None else default_config()
        h = C.c_void_p()
        _check(lib().a1mpc_create(C.byref(h), C.byref(self.cfg), device))
        self.h = h
        self.device = device
        self._ticks = weakref.WeakSet()

    @property
    def ftype(self):
        """element type of the hot-path boundary arrays (a1mpc_config::precision)"""
        return np.float32 if self.cfg.precision == 32 else np.float64

    def close(self):
        if self.h:
            for tick in list(getattr(self, "_ticks", ())):
                tick.close()
            lib().a1mpc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- hot path ----
    def _solve(self, fn, st, want_u=False, ext=None, warm_args=()):
        """one a1mpc_solve_batch* call on host arrays: ext = (sched [N,B] or None, normals [12,B] or None) for the _ext calls,
        warm_args = (warm, shift) for the _warm calls"""
        B = st["x0"].shape[1]
        N = self.cfg.horizon
        ft = self.ftype     # float32 arrays at the boundary when cfg.precision == 32
        a = {k: np.ascontiguousarray(st[k], dtype=(np.uint32 if k == "contact" else ft)) for k in ("x0", "rot", "foot", "ref", "contact")}
        f = np.zeros((12, B), dtype=ft); status = np.zeros(B, dtype=np.int32); iters = np.zeros(B, dtype=np.int32)
        u = np.zeros((12 * N, B), dtype=ft) if want_u else None
        inp = Inputs(_p(a["x0"]), _p(a["rot"]), _p(a["foot"]), _p(a["ref"]), _p(a["contact"]), B)
        out = Outputs(_p(f), _p(status), _p(iters), _p(u), B)
        ext_args = ()
        if ext is not None:
            sc = np.ascontiguousarray(ext[0], dtype=np.uint32) if ext[0] is not None else None
            nm = np.ascontiguousarray(ext[1], dtype=ft) if ext[1] is not None else None
            ext_args = (C.byref(InputsExt(_p(sc), _p(nm))),)
        _check(fn(self.h, B, C.byref(inp), *ext_args, C.byref(out), *warm_args))
        return (f, status, iters, u) if want_u else (f, status, iters)

    def solve(self, st, want_u=False):
        """host arrays in, host arrays out (H2D + kernels + D2H inside the call)"""
        return self._solve(lib().a1mpc_solve_batch, st, want_u)

    def warm_alloc(self, B):
        """device-resident warm-start state for B robots (no guess yet); free with a1mpc_device_free / Engine.dfree"""
        nbytes = lib().a1mpc_warm_bytes(self.h, B)
        p = self.dalloc(nbytes)
        _check(lib().a1mpc_warm_reset(self.h, p, B))
        return p

    def solve_warm(self, st, warm, shift=0):
        """a1mpc_solve_batch_warm: host arrays in/out, `warm` from warm_alloc (updated in place on the device)"""
        return self._solve(lib().a1mpc_solve_batch_warm, st, warm_args=(warm, int(shift)))

    def solve_ext(self, st, sched=None, normals=None, want_u=False):
        """BASELINE config 4 (extension): per-step contact schedule [N,B] and/or terrain normals [12,B]"""
        return self._solve(lib().a1mpc_solve_batch_ext, st, want_u, ext=(sched, normals))

    def solve_ext_warm(self, st, sched, normals, warm, shift=1, want_u=False):
        """a1mpc_solve_batch_ext_warm: solve_ext with the device-resident warm start (`warm` from warm_alloc, updated in place);
        shift = 1 for schedules that move one step per control tick (a1mpc_update_plan_batch)"""
        return self._solve(lib().a1mpc_solve_batch_ext_warm, st, want_u, ext=(sched, normals), warm_args=(warm, int(shift)))

    def solve_ptrs(self, B, inp, out):
        """raw a1mpc_solve_batch on caller-built Inputs/Outputs (host or device pointers)"""
        _check(lib().a1mpc_solve_batch(self.h, B, C.byref(inp), C.byref(out)))

    # ---- ConvexMpc parity members ----
    def build_qp(self, st):
        B = st["x0"].shape[1]
        N = self.cfg.horizon
        n, m = 12 * N, 20 * N
        a = {k: np.ascontiguousarray(st[k], dtype=(np.uint32 if k == "contact" else np.float64)) for k in ("x0", "rot", "foot", "ref", "contact")}
        H = np.zeros((B, n, n)); g = np.zeros((B, n)); lb = np.zeros((B, m)); ub = np.zeros((B, m))
        inp = Inputs(_p(a["x0"]), _p(a["rot"]), _p(a["foot"]), _p(a["ref"]), _p(a["contact"]), B)
        _check(lib().a1mpc_build_qp_batch(self.h, B, C.byref(inp), _p(H), _p(g), _p(lb), _p(ub)))
        return H, g, lb, ub

    def qp_mats(self, A_d, B_d_list, x0, x_d):
        A_d = np.ascontiguousarray(A_d, dtype=np.float64); B_d_list = np.ascontiguousarray(B_d_list, dtype=np.float64)
        x0 = np.ascontiguousarray(x0, dtype=np.float64); x_d = np.ascontiguousarray(x_d, dtype=np.float64)
        B = A_d.shape[0]
        n = 12 * self.cfg.horizon
        H = np.zeros((B, n, n)); g = np.zeros((B, n))
        _check(lib().a1mpc_qp_mats_batch(self.h, B, _p(A_d), _p(B_d_list), _p(x0), _p(x_d), _p(H), _p(g)))
        return H, g

    def qp_rollout(self, A_d, B_d_list, x0, x_d):
        """a1mpc_qp_rollout_batch: A_qp [B,13N,13], B_qp [B,13N,12N], H, g"""
        A_d = np.ascontiguousarray(A_d, dtype=np.float64); B_d_list = np.ascontiguousarray(B_d_list, dtype=np.float64)
        x0 = np.ascontiguousarray(x0, dtype=np.float64); x_d = np.ascontiguousarray(x_d, dtype=np.float64)
        B = A_d.shape[0]; N = self.cfg.horizon; n = 12 * N
        Aq = np.zeros((B, 13 * N, 13)); Bq = np.zeros((B, 13 * N, n)); H = np.zeros((B, n, n)); g = np.zeros((B, n))
        _check(lib().a1mpc_qp_rollout_batch(self.h, B, _p(A_d), _p(B_d_list), _p(x0), _p(x_d), _p(Aq), _p(Bq), _p(H), _p(g)))
        return Aq, Bq, H, g

    def solve_dense(self, H, g, contact):
        H = np.ascontiguousarray(H, dtype=np.float64); g = np.ascontiguousarray(g, dtype=np.float64)
        contact = np.ascontiguousarray(contact, dtype=np.uint32)
        B = H.shape[0]
        u = np.zeros((B, 12 * self.cfg.horizon)); status = np.zeros(B, dtype=np.int32)
        _check(lib().a1mpc_solve_dense_batch(self.h, B, _p(H), _p(g), _p(contact), _p(u), _p(status)))
        return u, status

    def grf_qp(self, root_acc, rot_z, rot, foot, contact):
        arrs = [np.ascontiguousarray(v, dtype=np.float64) for v in (root_acc, rot_z, rot, foot)]
        contact = np.ascontiguousarray(contact, dtype=np.uint32)
        B = arrs[0].shape[0]
        f = np.zeros((B, 12)); status = np.zeros(B, dtype=np.int32)
        _check(lib().a1mpc_grf_qp_batch(self.h, B, _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), _p(arrs[3]), _p(contact), _p(f), _p(status)))
        return f, status

    def stance_qp(self, x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, want_acc=False):
        """a1mpc_stance_qp_batch (compute_grf's QP branch from the controller state), batch-major host arrays: x0 [12,B], rot / rot_z [9,B],
        foot [12,B], contact [B], des [12,B] (root_euler_d, root_pos_d, root_lin_vel_d, root_ang_vel_d), kp_linear [3,B]; kd_linear,
        kp_angular, kd_angular [3] -> f_body [12,B], status [B] (, root_acc [6,B] when want_acc)"""
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x0, rot, rot_z, foot)]
        contact = np.ascontiguousarray(contact, dtype=np.uint32)
        d, kpl = np.ascontiguousarray(des, dtype=np.float64), np.ascontiguousarray(kp_linear, dtype=np.float64)
        g = [np.ascontiguousarray(v, dtype=np.float64) for v in (kd_linear, kp_angular, kd_angular)]
        B = contact.shape[0]
        f = np.zeros((12, B)); status = np.zeros(B, dtype=np.int32)
        acc = np.zeros((6, B)) if want_acc else None
        _check(lib().a1mpc_stance_qp_batch(self.h, B, B, *[_p(v) for v in a], _p(contact), _p(d), _p(kpl), *[_p(v) for v in g], _p(f), _p(status),
                                           _p(acc)))
        return (f, status, acc) if want_acc else (f, status)

    def stance_qp_ext(self, x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, normals, want_acc=False):
        """a1mpc_stance_qp_batch_ext: stance_qp with each stance foot's friction pyramid on its terrain normal, normals [12,B] (per foot, world
        frame, normalised by the engine) -> f_body [12,B], status [B] (, root_acc [6,B] when want_acc)"""
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x0, rot, rot_z, foot)]
        contact = np.ascontiguousarray(contact, dtype=np.uint32)
        d, kpl = np.ascontiguousarray(des, dtype=np.float64), np.ascontiguousarray(kp_linear, dtype=np.float64)
        g = [np.ascontiguousarray(v, dtype=np.float64) for v in (kd_linear, kp_angular, kd_angular)]
        nrm = np.ascontiguousarray(normals, dtype=np.float64)
        B = contact.shape[0]
        f = np.zeros((12, B)); status = np.zeros(B, dtype=np.int32)
        acc = np.zeros((6, B)) if want_acc else None
        _check(lib().a1mpc_stance_qp_batch_ext(self.h, B, B, *[_p(v) for v in a], _p(contact), _p(d), _p(kpl), *[_p(v) for v in g], _p(nrm), _p(f),
                                               _p(status), _p(acc)))
        return (f, status, acc) if want_acc else (f, status)

    def joint_torques(self, f_grf, f_kin, jac, contact, km_foot, torques_gravity, tau_prev=None):
        """batch-major SoA [12,B], [12,B], [36,B], [B] -> tau [12,B]"""
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (f_grf, f_kin, jac, km_foot, torques_gravity)]
        contact = np.ascontiguousarray(contact, dtype=np.uint32)
        B = a[0].shape[1]
        tau = np.zeros((12, B)) if tau_prev is None else np.ascontiguousarray(tau_prev, dtype=np.float64).copy()
        _check(lib().a1mpc_joint_torques_batch(self.h, B, _p(a[0]), _p(a[1]), _p(a[2]), _p(contact), _p(a[3]), _p(a[4]), _p(tau)))
        return tau

    def leg_kinematics(self, joint_pos, joint_vel, rot, rho_opt, rho_fix):
        """a1mpc_leg_kinematics_batch, host arrays: [12,B], [12,B], [9,B], rho_opt[12], rho_fix[20] ->
        foot_pos_rel [12,B], jac [36,B], foot_vel_rel [12,B], foot_pos_abs [12,B], foot_vel_abs [12,B]"""
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (joint_pos, joint_vel, rot, rho_opt, rho_fix)]
        B = a[0].shape[1]
        outs = [np.zeros((12, B)), np.zeros((36, B)), np.zeros((12, B)), np.zeros((12, B)), np.zeros((12, B))]
        _check(lib().a1mpc_leg_kinematics_batch(self.h, B, *[_p(v) for v in a], *[_p(o) for o in outs]))
        return outs

    def ekf_alloc(self, B):
        """device-resident filter state of B robots (342 doubles each: x[18], P[18,18])"""
        return self.dalloc(lib().a1mpc_ekf_bytes(B))

    def ekf_init(self, ekf, foot_pos_rel, rot):
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (foot_pos_rel, rot)]
        _check(lib().a1mpc_ekf_init_batch(self.h, a[0].shape[1], ekf, _p(a[0]), _p(a[1])))

    def ekf_update(self, ekf, dt, assume_flat_ground, movement_mode, imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel, foot_force):
        """a1mpc_ekf_update_batch, host arrays -> root_pos [3,B], root_lin_vel [3,B], estimated_contacts [B], status [B]"""
        mm = np.ascontiguousarray(movement_mode, dtype=np.uint32)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel, foot_force)]
        B = mm.shape[0]
        pos = np.zeros((3, B)); vel = np.zeros((3, B)); ec = np.zeros(B, dtype=np.uint32); status = np.full(B, -7, dtype=np.int32)
        _check(lib().a1mpc_ekf_update_batch(self.h, B, ekf, C.c_double(dt), int(assume_flat_ground), _p(mm), *[_p(v) for v in a],
                                            _p(pos), _p(vel), _p(ec), _p(status)))
        return pos, vel, ec, status

    def ekf_state(self, ekf, B):
        """copy of the device-resident filter state: x [B,18], P [B,18,18]"""
        buf = np.zeros((B, 342))
        _check(lib().a1mpc_memcpy_d2h(self.h, _p(buf), ekf, buf.nbytes))
        _check(lib().a1mpc_sync(self.h))
        return buf[:, :18].copy(), buf[:, 18:].reshape(B, 18, 18).copy()

    def swing_alloc(self, B):
        """device-resident swing-leg / terrain controller state of B robots (a1mpc_swing_bytes), initialised by a1mpc_swing_init_batch;
        bound to this B"""
        p = self.dalloc(lib().a1mpc_swing_bytes(B))
        self.swing_init(p, B)
        return p

    def swing_init(self, swing, B):
        """a1mpc_swing_init_batch: A1CtrlStates::reset() values and empty filters"""
        _check(lib().a1mpc_swing_init_batch(self.h, B, swing))

    def swing_legs(self, gp, kp_foot, kd_foot, swing, dt, gait_counter, plan_contacts, rot_z, foot_pos_abs, foot_pos_target_rel, foot_force):
        """a1mpc_swing_legs_batch (generate_swing_legs_ctrl), host arrays: gait_counter [4,B], plan_contacts [B], rot_z [9,B],
        foot_pos_abs / foot_pos_target_rel [12,B], foot_force [4,B]; kp_foot, kd_foot [12] leg-major ->
        f_kin [12,B], contacts [B], foot_pos_cur [12,B], foot_pos_recent_contact [12,B]"""
        kp, kd, gc = [np.ascontiguousarray(v, dtype=np.float64) for v in (kp_foot, kd_foot, gait_counter)]
        pc = np.ascontiguousarray(plan_contacts, dtype=np.uint32)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (rot_z, foot_pos_abs, foot_pos_target_rel, foot_force)]
        B = pc.shape[0]
        fk = np.zeros((12, B)); con = np.zeros(B, dtype=np.uint32); cur = np.zeros((12, B)); rc = np.zeros((12, B))
        _check(lib().a1mpc_swing_legs_batch(self.h, B, C.byref(gp), _p(kp), _p(kd), swing, C.c_double(dt), _p(gc), _p(pc), *[_p(v) for v in a],
                                            _p(fk), _p(con), _p(cur), _p(rc)))
        return fk, con, cur, rc

    def terrain_pitch(self, swing, use_terrain_adapt, root_pos, ref=None):
        """a1mpc_terrain_pitch_batch, host arrays: root_pos [3,B]; ref [9,B] (a1mpc_inputs.ref layout) gets row 1 in place when
        use_terrain_adapt -> terrain_pitch [B]"""
        pos = np.ascontiguousarray(root_pos, dtype=np.float64)
        B = pos.shape[1]
        if ref is not None and not (ref.dtype == np.float64 and ref.flags["C_CONTIGUOUS"]):
            raise A1MpcError("ref must be a C-contiguous float64 array (written in place)")
        pitch = np.zeros(B)
        _check(lib().a1mpc_terrain_pitch_batch(self.h, B, swing, int(use_terrain_adapt), _p(pos), _p(ref), ref.shape[1] if ref is not None else B,
                                               _p(pitch)))
        return pitch

    def terrain_normals(self, swing, use_terrain_adapt, root_pos, ref=None):
        """a1mpc_terrain_normals_batch, host arrays: terrain_pitch plus the walking surface's unit normal -> (terrain_pitch [B],
        normals [12,B], the same for all four feet)"""
        pos = np.ascontiguousarray(root_pos, dtype=np.float64)
        B = pos.shape[1]
        if ref is not None and not (ref.dtype == np.float64 and ref.flags["C_CONTIGUOUS"]):
            raise A1MpcError("ref must be a C-contiguous float64 array (written in place)")
        pitch = np.zeros(B)
        normals = np.zeros((12, B))
        _check(lib().a1mpc_terrain_normals_batch(self.h, B, swing, int(use_terrain_adapt), _p(pos), _p(ref), ref.shape[1] if ref is not None else B,
                                                 _p(pitch), _p(normals)))
        return pitch, normals

    def surface_normals(self, swing, root_pos):
        """a1mpc_surface_normals_batch, host arrays: the walking surface's unit normal of terrain_normals without the terrain stage (the
        swing state is only read) -> normals [12,B], the same for all four feet"""
        pos = np.ascontiguousarray(root_pos, dtype=np.float64)
        B = pos.shape[1]
        normals = np.zeros((12, B))
        _check(lib().a1mpc_surface_normals_batch(self.h, B, swing, _p(pos), _p(normals)))
        return normals

    def plan_forces(self, rot, u_full, step, f_body=None):
        """a1mpc_plan_forces_batch on host arrays: rot [9][B], u_full [12N][B], step [B] -> f_body [12][B] (a copy of the given f_body, or
        zeros, where step is 0; R^T of plan step `step` where 0 < step < N; zero forces where step >= N)"""
        B = np.shape(step)[0]
        r = np.ascontiguousarray(rot, dtype=np.float64); u = np.ascontiguousarray(u_full, dtype=np.float64)
        s = np.ascontiguousarray(step, dtype=np.uint32)
        f = np.array(f_body, dtype=np.float64, order="C") if f_body is not None else np.zeros((12, B))
        if r.shape != (9, B) or u.shape != (12 * self.cfg.horizon, B) or f.shape != (12, B):
            raise ValueError("rot must be [9][B], u_full [12N][B] and f_body [12][B]")
        _check(lib().a1mpc_plan_forces_batch(self.h, B, _p(r), _p(u), _p(s), _p(f)))
        return f

    def imu_alloc(self, B):
        """device-resident IMU filter state of B robots (a1mpc_imu_bytes), initialised by a1mpc_imu_init_batch; bound to this B"""
        p = self.dalloc(lib().a1mpc_imu_bytes(B))
        self.imu_init(p, B)
        return p

    def imu_init(self, imu, B):
        """a1mpc_imu_init_batch: six empty MovingWindowFilter(5)"""
        _check(lib().a1mpc_imu_init_batch(self.h, B, imu))

    def orientation(self, quat, gyro, acc=None, imu=None):
        """a1mpc_orientation_batch, host arrays: quat [4,B] (w, x, y, z), gyro / acc [3,B]; imu = the filter state or None (unfiltered) ->
        dict rot [9,B], rot_z [9,B], euler [3,B], ang_vel [3,B] (x0 rows 0-2 and 6-8), imu_acc [3,B] (None without acc), imu_ang_vel [3,B]"""
        q, g = [np.ascontiguousarray(v, dtype=np.float64) for v in (quat, gyro)]
        a = np.ascontiguousarray(acc, dtype=np.float64) if acc is not None else None
        B = q.shape[1]
        x0 = np.zeros((12, B)); rot = np.zeros((9, B)); rz = np.zeros((9, B)); ia = np.zeros((3, B)) if a is not None else None; ig = np.zeros((3, B))
        _check(lib().a1mpc_orientation_batch(self.h, B, _p(q), _p(g), _p(a), imu, _p(rot), _p(rz), _p(x0), B, _p(ia), _p(ig)))
        return dict(rot=rot, rot_z=rz, euler=x0[0:3].copy(), ang_vel=x0[6:9].copy(), imu_acc=ia, imu_ang_vel=ig)

    def command_alloc(self, B, params=None, ref=None):
        """device-resident command state of B robots (a1mpc_command_bytes), initialised by a1mpc_command_init_batch from params
        (default_command_params()); ref [9,B] (host, written in place) gets the reset rows.  Bound to this B"""
        p = self.dalloc(lib().a1mpc_command_bytes(B))
        self.command_init(p, B, params, ref)
        return p

    def command_init(self, cmd_state, B, params=None, ref=None):
        """a1mpc_command_init_batch"""
        cp = params if params is not None else default_command_params()
        if ref is not None and not (ref.dtype == np.float64 and ref.flags["C_CONTIGUOUS"]):
            raise A1MpcError("ref must be a C-contiguous float64 array (written in place)")
        _check(lib().a1mpc_command_init_batch(self.h, B, cmd_state, C.byref(cp), _p(ref), ref.shape[1] if ref is not None else B))

    def command(self, cmd_state, dt, cmd, root_pos, ref=None):
        """a1mpc_command_batch, host arrays: cmd [7,B] (velx, vely, velz, roll / pitch / yaw rate, toggle), root_pos [3,B]; ref [9,B]
        (a1mpc_inputs.ref layout, in / out in place: row 1 is this tick's starting root_euler_d[1]) ->
        movement_mode [B], kp_linear [3,B], des [12,B] (a1mpc_stance_qp_batch layout)"""
        c, pos = [np.ascontiguousarray(v, dtype=np.float64) for v in (cmd, root_pos)]
        B = c.shape[1]
        if ref is not None and not (ref.dtype == np.float64 and ref.flags["C_CONTIGUOUS"]):
            raise A1MpcError("ref must be a C-contiguous float64 array (written in place)")
        mode = np.zeros(B, dtype=np.uint32); kp = np.zeros((3, B)); des = np.zeros((12, B))
        _check(lib().a1mpc_command_batch(self.h, B, cmd_state, C.c_double(dt), _p(c), _p(pos), B, _p(mode), _p(kp), _p(ref),
                                         ref.shape[1] if ref is not None else B, _p(des), B))
        return mode, kp, des

    def update_plan(self, gp, gait_counter, gait_counter_speed, movement_mode, lin_vel, lin_vel_d, rot_z, rot, root_pos):
        """A1RobotControl::update_plan batched; returns new gait_counter [4,B], plan_contacts [B], contact_sched [N,B],
        foot_pos_target_rel/abs/world [12,B]"""
        gc = np.ascontiguousarray(gait_counter, dtype=np.float64).copy()
        B = gc.shape[1]
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (gait_counter_speed, lin_vel, lin_vel_d, rot_z, rot, root_pos)]
        mode = np.ascontiguousarray(movement_mode, dtype=np.uint32)
        plan = np.zeros(B, dtype=np.uint32); sched = np.zeros((gp.horizon, B), dtype=np.uint32)
        trel = np.zeros((12, B)); tabs = np.zeros((12, B)); tw = np.zeros((12, B))
        _check(lib().a1mpc_update_plan_batch(self.h, B, C.byref(gp), _p(gc), _p(a[0]), _p(mode), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]),
                                             _p(plan), _p(sched), _p(trel), _p(tabs), _p(tw)))
        return gc, plan, sched, trel, tabs, tw

    def update_plan_gait(self, gp, gait, gait_counter, gait_counter_speed, movement_mode, lin_vel, lin_vel_d, rot_z, rot, root_pos):
        """a1mpc_update_plan_gait_batch: update_plan with each robot's gait row, gait [6,B]; returns what update_plan returns"""
        g = np.ascontiguousarray(gait, dtype=np.float64)
        gc = np.ascontiguousarray(gait_counter, dtype=np.float64).copy()
        B = gc.shape[1]
        if g.shape != (6, B):
            raise ValueError("gait rows must have shape (6, %d)" % B)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (gait_counter_speed, lin_vel, lin_vel_d, rot_z, rot, root_pos)]
        mode = np.ascontiguousarray(movement_mode, dtype=np.uint32)
        plan = np.zeros(B, dtype=np.uint32); sched = np.zeros((gp.horizon, B), dtype=np.uint32)
        trel = np.zeros((12, B)); tabs = np.zeros((12, B)); tw = np.zeros((12, B))
        _check(lib().a1mpc_update_plan_gait_batch(self.h, B, C.byref(gp), _p(g), _p(gc), _p(a[0]), _p(mode), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]),
                                                  _p(a[5]), _p(plan), _p(sched), _p(trel), _p(tabs), _p(tw)))
        return gc, plan, sched, trel, tabs, tw

    def swing_legs_gait(self, gp, gait, kp_foot, kd_foot, swing, dt, gait_counter, plan_contacts, rot_z, foot_pos_abs, foot_pos_target_rel, foot_force):
        """a1mpc_swing_legs_gait_batch: swing_legs with each robot's gait row, gait [6,B]; returns what swing_legs returns"""
        g = np.ascontiguousarray(gait, dtype=np.float64)
        kp, kd, gc = [np.ascontiguousarray(v, dtype=np.float64) for v in (kp_foot, kd_foot, gait_counter)]
        pc = np.ascontiguousarray(plan_contacts, dtype=np.uint32)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (rot_z, foot_pos_abs, foot_pos_target_rel, foot_force)]
        B = pc.shape[0]
        if g.shape != (6, B):
            raise ValueError("gait rows must have shape (6, %d)" % B)
        fk = np.zeros((12, B)); con = np.zeros(B, dtype=np.uint32); cur = np.zeros((12, B)); rc = np.zeros((12, B))
        _check(lib().a1mpc_swing_legs_gait_batch(self.h, B, C.byref(gp), _p(g), _p(kp), _p(kd), swing, C.c_double(dt), _p(gc), _p(pc),
                                                 *[_p(v) for v in a], _p(fk), _p(con), _p(cur), _p(rc)))
        return fk, con, cur, rc

    # ---- memory / timing helpers ----
    def dalloc(self, nbytes):
        p = C.c_void_p()
        _check(lib().a1mpc_device_alloc(self.h, nbytes, C.byref(p)))
        return p

    def halloc(self, nbytes):
        p = C.c_void_p()
        _check(lib().a1mpc_host_alloc(self.h, nbytes, C.byref(p)))
        return p

    def pinned_array(self, shape, dtype):
        """numpy view over pinned host memory (kept alive by the returned array's base object)"""
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = self.halloc(max(nbytes, 8))
        buf = (C.c_char * nbytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype).reshape(shape)
        return arr

    def sync(self):
        _check(lib().a1mpc_sync(self.h))

    def event(self):
        e = C.c_void_p()
        _check(lib().a1mpc_event_create(self.h, C.byref(e)))
        return e

    def record(self, ev):
        _check(lib().a1mpc_event_record(self.h, ev))

    def elapsed_ms(self, e0, e1):
        ms = C.c_float()
        _check(lib().a1mpc_event_elapsed_ms(self.h, e0, e1, C.byref(ms)))
        return float(ms.value)

    def launches(self):
        return int(lib().a1mpc_launch_count(self.h))

    def fp64_peak_tflops(self):
        v = C.c_double()
        _check(lib().a1mpc_measure_fp64_peak(self.h, C.byref(v)))
        return float(v.value)

    def profile_begin(self, max_calls):
        _check(lib().a1mpc_profile_begin(self.h, max_calls))

    def profile_end(self):
        ms = np.zeros(4); n = C.c_int()
        _check(lib().a1mpc_profile_end(self.h, _p(ms), C.byref(n)))
        return ms, int(n.value)

    def nccl_init(self, nranks, rank, uid_bytes):
        buf = C.create_string_buffer(bytes(uid_bytes), 128)
        _check(lib().a1mpc_nccl_init(self.h, nranks, rank, buf))

    def allgather_forces(self, f_local_ptr, f_all_ptr, B_local):
        _check(lib().a1mpc_allgather_forces(self.h, f_local_ptr, f_all_ptr, B_local))

    # ---- fused final collect over peer memory (one process per GPU) ----
    def peer_gather_create(self, nranks, rank, B_local):
        """allocates this rank's gathered buffer; returns the 64-byte CUDA IPC handle to hand to the other ranks"""
        hd = (C.c_char * 64)()
        _check(lib().a1mpc_peer_gather_create(self.h, int(nranks), int(rank), int(B_local), hd))
        return bytes(hd.raw)

    def peer_gather_connect(self, handles):
        """handles: the ranks' 64-byte handles in rank order (list of bytes)"""
        blob = b"".join(handles)
        _check(lib().a1mpc_peer_gather_connect(self.h, C.c_char_p(blob)))

    def peer_gather_buffer(self):
        p = C.c_void_p()
        _check(lib().a1mpc_peer_gather_buffer(self.h, C.byref(p)))
        return p

    def peer_gather_wait(self):
        _check(lib().a1mpc_peer_gather_wait(self.h))

    def peer_gather_status(self):
        v = C.c_int()
        _check(lib().a1mpc_peer_gather_status(self.h, C.byref(v)))
        return v.value

    def peer_gather_destroy(self):
        _check(lib().a1mpc_peer_gather_destroy(self.h))

    def flush_l2(self):
        _check(lib().a1mpc_flush_l2(self.h))


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    _check(lib().a1mpc_nccl_unique_id(buf))
    return bytes(buf.raw)
