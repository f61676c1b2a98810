"""CPU test of the multi-rate tick's entry points (a1mpc_tick_set_mpc_period, a1mpc_plan_forces_batch) and their bindings: the prototypes and
constants in include/a1mpc.h, the ctypes argument types, Tick.set_mpc_period and Engine.plan_forces marshalling their arguments down to the C
call (which rejects the NULL tick or handle with A1MPC_EINVAL), and the shape errors Engine.plan_forces raises before any device work."""
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
    assert re.search(r"int\s+a1mpc_tick_set_mpc_period\(a1mpc_tick\* t, int period, int playback\);", hdr)
    assert re.search(r"int\s+a1mpc_plan_forces_batch\(a1mpc_handle\* h, int B, const double\* rot, const double\* u_full, "
                     r"const uint32_t\* step, double\* f_body\);", hdr)
    consts = dict(re.findall(r"#define\s+A1MPC_PLAYBACK_(\w+)\s+(\d+)", hdr))
    assert consts == {"HOLD": "0", "PLAN": "1"}
    assert (a1.PLAYBACK_HOLD, a1.PLAYBACK_PLAN) == (0, 1)
    for name in ("a1mpc_tick_set_mpc_period", "a1mpc_plan_forces_batch"):
        assert name in a1.EXPORTS
    L = a1.lib()
    assert L.a1mpc_tick_set_mpc_period.argtypes == [C.c_void_p, C.c_int, C.c_int]
    assert L.a1mpc_plan_forces_batch.argtypes == [C.c_void_p, C.c_int] + [C.c_void_p] * 4


def test_null_tick_and_handle_are_rejected(a1):
    L = a1.lib()
    assert L.a1mpc_tick_set_mpc_period(None, 2, a1.PLAYBACK_PLAN) == -1 and b"null argument" in L.a1mpc_last_error()
    rot, u, step, f = np.zeros((9, 4)), np.zeros((120, 4)), np.zeros(4, np.uint32), np.zeros((12, 4))
    assert L.a1mpc_plan_forces_batch(None, 4, rot.ctypes.data, u.ctypes.data, step.ctypes.data, f.ctypes.data) == -1
    assert b"null argument" in L.a1mpc_last_error()


def _null_engine(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    return eng


def test_bindings_marshal_their_arguments(a1):
    B = 4
    eng = _null_engine(a1)
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, a1.default_tick_params(), None
    for args in ((2,), (4, a1.PLAYBACK_HOLD), (10, a1.PLAYBACK_PLAN), (np.int64(3),)):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.set_mpc_period(*args)
    N = eng.cfg.horizon
    for f_body in (None, np.ones((12, B))):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            eng.plan_forces(np.zeros((9, B)), np.zeros((12 * N, B)), np.arange(B), f_body)


@pytest.mark.parametrize("bad", ["rot", "u_full", "f_body"])
def test_plan_forces_rejects_malformed_arrays(a1, bad):
    B = 4
    eng = _null_engine(a1)
    N = eng.cfg.horizon
    args = dict(rot=np.zeros((9, B)), u_full=np.zeros((12 * N, B)), step=np.zeros(B, np.uint32), f_body=np.zeros((12, B)))
    args[bad] = np.zeros((args[bad].shape[0] + 1, B))
    with pytest.raises(ValueError, match="u_full"):
        eng.plan_forces(**args)
