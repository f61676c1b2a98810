"""CPU test of the bindings of the orientation / command entry points: with a NULL handle every C entry point must reject the call with
A1MPC_EINVAL after ctypes has converted every argument against the declared prototype; the argument checks that need no device; the
state sizes; and the row offsets of the ld layouts the calls share with a1mpc_inputs and a1mpc_stance_qp_batch."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_command_bindings_marshal_their_arguments(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    B = 4
    null = C.c_void_p(0)
    rng = np.random.default_rng(0)
    r = lambda *s: rng.standard_normal(s)
    calls = [
        lambda: eng.imu_alloc(B),
        lambda: eng.imu_init(null, B),
        lambda: eng.orientation(r(4, B), r(3, B)),
        lambda: eng.orientation(r(4, B), r(3, B), r(3, B), null),
        lambda: eng.command_alloc(B),
        lambda: eng.command_init(null, B, a1.default_command_params(a1.VARIANT_HARDWARE), np.zeros((9, B))),
        lambda: eng.command(null, 0.0025, r(7, B), r(3, B)),
        lambda: eng.command(null, 0.0025, r(7, B), r(3, B), np.zeros((9, B))),
    ]
    for call in calls:
        with pytest.raises(a1.A1MpcError, match="null argument"):
            call()
    eng.h = None


def test_sizes_and_argument_checks(a1):
    L = a1.lib()
    B = 8
    assert L.a1mpc_imu_bytes(B) == B * 54 * 8 and L.a1mpc_imu_bytes(0) == 0 and L.a1mpc_imu_bytes(-1) == 0
    assert L.a1mpc_command_bytes(B) == B * 19 * 8 and L.a1mpc_command_bytes(0) == 0
    assert L.a1mpc_imu_init_batch(None, B, None) == -1
    assert L.a1mpc_orientation_batch(None, B, None, None, None, None, None, None, None, B, None, None) == -1
    cp = a1.default_command_params()
    assert L.a1mpc_command_init_batch(None, B, None, C.byref(cp), None, B) == -1
    assert L.a1mpc_command_batch(None, B, None, 0.0025, None, None, B, None, None, None, B, None, B) == -1
    assert b"null argument" in L.a1mpc_last_error()


def test_default_command_params(a1):
    h = {a1.VARIANT_GAZEBO: 0.3, a1.VARIANT_HARDWARE: 0.12, a1.VARIANT_ISAAC: 0.32}
    for v, h0 in h.items():
        cp = a1.default_command_params(v)
        assert cp.variant == v and cp.body_height == h0 and (cp.body_height_min, cp.body_height_max) == (0.1, 0.32)
        assert list(cp.kp_linear) == [120.0, 120.0, 500.0] and list(cp.kp_linear_lock) == [120.0, 120.0]
    assert C.sizeof(a1.CommandParams) == 8 + 8 * 8


def test_ld_row_offsets():
    """the rows the calls read and write inside the arrays of the other stages, with a leading dimension ld > B"""
    B, ld = 5, 9
    x0 = np.arange(12 * ld, dtype=np.float64).reshape(12, ld)
    base = x0.ctypes.data
    # orientation: x0 rows 0-2 (root_euler) at x0, rows 6-8 (root_ang_vel) at x0 + 6 ld; command: root_pos at x0 + 3 ld
    assert np.frombuffer((C.c_double * B).from_address(base + 6 * ld * 8), dtype=np.float64).tolist() == x0[6, :B].tolist()
    assert np.frombuffer((C.c_double * B).from_address(base + 3 * ld * 8), dtype=np.float64).tolist() == x0[3, :B].tolist()
    # ref: root_lin_vel_d at ref + 5 ref_ld (the lin_vel_d input of a1mpc_update_plan_batch); des: root_lin_vel_d at rows 6-8
    ref = np.arange(9 * ld, dtype=np.float64).reshape(9, ld)
    assert np.frombuffer((C.c_double * (3 * ld)).from_address(ref.ctypes.data + 5 * ld * 8), dtype=np.float64).reshape(3, ld).tolist() == ref[5:8].tolist()
