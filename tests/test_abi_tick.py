"""CPU test of the tick bindings (a1mpc_default_tick_params, a1mpc_tick_*): every new prototype marshals its arguments and a NULL handle or
tick is rejected with A1MPC_EINVAL; the ctypes structs have the C layout of include/a1mpc.h; and the default parameters are the reference's
launch values for the three adapters in both stance modes."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_tick_bindings_marshal_their_arguments(a1):
    L = a1.lib()
    B = 4
    tp = a1.default_tick_params()
    t = C.c_void_p()
    assert L.a1mpc_tick_create(None, B, C.byref(tp), C.byref(t)) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_tick_reset(None) == -1 and b"null argument" in L.a1mpc_last_error()
    ins, outs = a1.TickInputs(), a1.TickOutputs()
    assert L.a1mpc_tick_run(None, 0.0025, C.byref(ins), C.byref(outs)) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_tick_destroy(None) == 0
    assert L.a1mpc_default_tick_params(0, 1, None) == -1 and b"null argument" in L.a1mpc_last_error()
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    with pytest.raises(a1.A1MpcError, match="null argument"):
        a1.Tick(eng, B, tp)
    # the Python wrappers marshal host arrays into the structs the C call takes
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, tp, None
    r = lambda *s: np.zeros(s)
    with pytest.raises(a1.A1MpcError, match="null argument"):
        tick.run(0.0025, r(4, B), r(3, B), r(3, B), r(12, B), r(12, B), r(4, B), r(7, B), r(4, B))
    with pytest.raises(ValueError):
        tick.run(0.0025, r(4, B + 1), r(3, B), r(3, B), r(12, B), r(12, B), r(4, B), r(7, B), r(4, B))
    for call in (tick.reset, lambda: tick.run_ptrs(0.0025, ins, outs)):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            call()


def test_struct_layouts(a1):
    # a1mpc_gait_params: 17 doubles + int (padded to 144); a1mpc_command_params: int + 8 doubles (72)
    assert C.sizeof(a1.GaitParams) == 144 and C.sizeof(a1.CommandParams) == 72
    T = a1.TickParams
    assert (T.mode.offset, T.use_terrain_adapt.offset, T.assume_flat_ground.offset) == (0, 4, 8)
    assert T.gait.offset == 16 and T.command.offset == 16 + 144 and T.rho_opt.offset == 16 + 144 + 72
    assert C.sizeof(T) == 232 + 8 * (12 + 20 + 12 + 12 + 3 + 12 + 3 + 3 + 3)
    assert C.sizeof(a1.TickInputs) == 8 * 8 and C.sizeof(a1.TickOutputs) == 7 * 8
    assert [f[0] for f in a1.TickInputs._fields_] == ["quat", "gyro", "acc", "joint_pos", "joint_vel", "foot_force", "cmd", "gait_counter_speed"]
    assert [f[0] for f in a1.TickOutputs._fields_] == ["tau", "f_body", "status", "contacts", "movement_mode", "x0", "ref"]


# config/<variant>_a1_<mode>.yaml of the reference: a1_kp_foot_*, a1_kd_foot_*, a1_km_foot_*, a1_default_foot_pos_* (FL x, z) and, in QP mode,
# a1_kp_linear_*, a1_kd_linear_*, a1_kp_angular_*, a1_kd_angular_*
YAML = {
    ("gazebo", "mpc"): dict(kp=(200, 200, 150), kd=(10, 10, 5), km=(0.1,) * 3, fx=0.17, fz=-0.35),
    ("gazebo", "qp"): dict(kp=(300, 400, 400), kd=(8, 8, 8), km=(0.1,) * 3, fx=0.17, fz=-0.35, kpl=(100, 100, 300), kdl=(70, 70, 120),
                           kpa=(150, 150, 1), kda=(4.5, 4.5, 30)),
    ("hardware", "mpc"): dict(kp=(120, 120, 80), kd=(6, 6, 5), km=(0.1,) * 3, fx=0.17, fz=-0.3),
    ("hardware", "qp"): dict(kp=(260, 260, 350), kd=(6, 6, 5), km=(0.1,) * 3, fx=0.17, fz=-0.33, kpl=(400, 400, 1500), kdl=(300, 200, 120),
                             kpa=(40, 40, 10), kda=(1, 1, 0.5)),
    ("isaac", "mpc"): dict(kp=(3250, 3250, 4000), kd=(5, 5, 5), km=(0.5,) * 3, fx=0.24, fz=-0.35),
    ("isaac", "qp"): dict(kp=(4250, 4250, 3000), kd=(0, 0, 0), km=(0.5,) * 3, fx=0.25, fz=-0.33, kpl=(1450, 1450, 3800), kdl=(2600, 2600, 0),
                          kpa=(420, 420, 150), kda=(0, 0, 560)),
}


@pytest.mark.parametrize("variant", ["gazebo", "hardware", "isaac"])
@pytest.mark.parametrize("mode", ["qp", "mpc"])
def test_default_tick_params(a1, variant, mode):
    v = dict(gazebo=a1.VARIANT_GAZEBO, hardware=a1.VARIANT_HARDWARE, isaac=a1.VARIANT_ISAAC)[variant]
    m = a1.TICK_MPC if mode == "mpc" else a1.TICK_QP
    tp = a1.default_tick_params(v, m)
    y = YAML[(variant, mode)]
    assert tp.mode == m and tp.command.variant == v
    assert tp.use_terrain_adapt == (0 if (variant, mode) == ("isaac", "mpc") else 1)   # isaac_a1_mpc.yaml:3; A1CtrlStates.h:137
    assert tp.assume_flat_ground == 1                                                  # A1BasicEKF.cpp:40
    g = tp.gait
    assert (g.counter_per_gait, g.counter_per_swing, g.control_dt, g.foot_delta_x_limit, g.foot_delta_y_limit) == (240.0, 120.0, 0.0025, 0.1, 0.1)
    fx, fz = y["fx"], y["fz"]
    assert list(g.default_foot_pos) == [fx, fx, -0.17, -0.17, 0.15, -0.15, 0.15, -0.15, fz, fz, fz, fz]
    assert list(tp.kp_foot) == list(y["kp"]) * 4 and list(tp.kd_foot) == list(y["kd"]) * 4 and tuple(tp.km_foot) == y["km"]
    assert list(tp.torques_gravity) == [0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0]   # A1CtrlStates.h:129
    c = tp.command
    assert c.body_height == dict(gazebo=0.3, hardware=0.12, isaac=0.32)[variant] and (c.body_height_min, c.body_height_max) == (0.1, 0.32)
    kpl = y.get("kpl", (120, 120, 500))                                                # A1CtrlStates.h:273-275 without the yaml keys
    assert tuple(c.kp_linear) == kpl and tuple(c.kp_linear_lock) == kpl[:2]
    if mode == "qp":
        assert (tuple(tp.kd_linear), tuple(tp.kp_angular), tuple(tp.kd_angular)) == (y["kdl"], y["kpa"], y["kda"])
    upper = dict(gazebo=0.21, hardware=0.20, isaac=0.22)[variant]
    lower = 0.20 if variant == "hardware" else 0.21
    rf = np.array(tp.rho_fix).reshape(4, 5)
    assert np.array_equal(rf[:, 0], [0.1805, 0.1805, -0.1805, -0.1805]) and np.array_equal(rf[:, 1], [0.047, -0.047, 0.047, -0.047])
    assert np.array_equal(rf[:, 2], [0.0838, -0.0838, 0.0838, -0.0838]) and (rf[:, 3] == upper).all() and (rf[:, 4] == lower).all()
    assert list(tp.rho_opt) == [0.0] * 12


def test_default_tick_params_rejects_unknown_values(a1):
    L = a1.lib()
    tp = a1.TickParams()
    assert L.a1mpc_default_tick_params(3, a1.TICK_MPC, C.byref(tp)) == -1 and b"variant" in L.a1mpc_last_error()
    assert L.a1mpc_default_tick_params(a1.VARIANT_GAZEBO, 2, C.byref(tp)) == -1 and b"mode" in L.a1mpc_last_error()
