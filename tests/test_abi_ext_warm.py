"""CPU test of the binding of a1mpc_solve_batch_ext_warm: with a NULL handle the C entry point must reject the call with
A1MPC_EINVAL after ctypes has converted every argument against the declared prototype."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_solve_ext_warm_binding_marshals_its_arguments(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    B = 4
    st = a1.gen_states(B, 2, 1)
    sched, normals = a1.gen_schedule(B, 10, 4, 1)
    for kw in ({}, {"shift": 0, "want_u": True}):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            eng.solve_ext_warm(st, sched, normals, C.c_void_p(0), **kw)
    with pytest.raises(a1.A1MpcError):
        eng.solve_ext_warm(st, None, None, C.c_void_p(0))
    assert a1.lib().a1mpc_solve_batch_ext_warm(None, B, None, None, None, None, 1) == -1
    eng.h = None
