"""CPU test of the per-robot gait entry points (a1mpc_gait_row, a1mpc_update_plan_gait_batch, a1mpc_swing_legs_gait_batch,
a1mpc_tick_set_gaits) and their bindings: the prototypes and constants in include/a1mpc.h, the ctypes argument types, the bindings
marshalling their arguments down to the C call (which rejects the NULL tick or handle with A1MPC_EINVAL), and the shape errors raised
before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_prototypes_constants_and_exports(a1):
    hdr = open(os.path.join(ROOT, "include", "a1mpc.h")).read()
    assert re.search(r"int\s+a1mpc_gait_row\(int gait_type, double row\[6\]\);", hdr)
    assert re.search(r"int\s+a1mpc_tick_set_gaits\(a1mpc_tick\* t, const double\* gait\);", hdr)
    assert re.search(r"int\s+a1mpc_update_plan_gait_batch\(a1mpc_handle\* h, int B, const a1mpc_gait_params\* gp, const double\* gait, double\* gait_counter,", hdr)
    assert re.search(r"int\s+a1mpc_swing_legs_gait_batch\(a1mpc_handle\* h, int B, const a1mpc_gait_params\* gp, const double\* gait, const double\* kp_foot,", hdr)
    consts = dict(re.findall(r"#define\s+A1MPC_GAIT_(\w+)\s+(\d+)", hdr))
    assert consts == {"TROT": "1", "PACE": "2", "BOUND": "3", "PRONK": "4", "WALK": "5"}
    for name in ("a1mpc_gait_row", "a1mpc_tick_set_gaits", "a1mpc_update_plan_gait_batch", "a1mpc_swing_legs_gait_batch"):
        assert name in a1.EXPORTS and hasattr(a1.lib(), name)
    L = a1.lib()
    assert L.a1mpc_tick_set_gaits.argtypes == [C.c_void_p, C.c_void_p]
    assert L.a1mpc_gait_row.argtypes == [C.c_int, C.c_void_p]
    assert L.a1mpc_update_plan_gait_batch.argtypes[3:] == [C.c_void_p] * 14
    assert L.a1mpc_swing_legs_gait_batch.argtypes[7] == C.c_double and len(L.a1mpc_swing_legs_gait_batch.argtypes) == 18


def test_null_arguments_are_rejected(a1):
    L = a1.lib()
    assert L.a1mpc_tick_set_gaits(None, None) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_gait_row(1, None) == -1 and b"null argument" in L.a1mpc_last_error()
    gp = a1.default_tick_params().gait
    z = np.zeros((12, 4))
    assert L.a1mpc_update_plan_gait_batch(None, 4, C.byref(gp), *([z.ctypes.data] * 14)) == -1
    assert L.a1mpc_swing_legs_gait_batch(None, 4, C.byref(gp), z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, 0.0025,
                                         *([z.ctypes.data] * 10)) == -1
    assert b"null argument" in L.a1mpc_last_error()


def test_bindings_marshal_their_arguments(a1):
    B = 5
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, a1.default_tick_params(), None
    rows = np.stack([a1.gait_row(1 + b) for b in range(B)], axis=1)
    for r in (rows, None):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.set_gaits(r)
    with pytest.raises(ValueError, match="shape"):
        tick.set_gaits(rows[:, :3])
    gp = a1.default_tick_params().gait
    z = lambda r: np.zeros((r, B))
    with pytest.raises(a1.A1MpcError, match="null argument"):
        eng.update_plan_gait(gp, rows, z(4), z(4), np.zeros(B), z(3), z(3), z(9), z(9), z(3))
    with pytest.raises(ValueError, match="shape"):
        eng.update_plan_gait(gp, rows[:5], z(4), z(4), np.zeros(B), z(3), z(3), z(9), z(9), z(3))
    with pytest.raises(a1.A1MpcError, match="null argument"):
        eng.swing_legs_gait(gp, rows, np.zeros(12), np.zeros(12), None, 0.0025, z(4), np.zeros(B), z(9), z(12), z(12), z(4))
