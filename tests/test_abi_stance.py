"""CPU test of the binding of a1mpc_stance_qp_batch: with a NULL handle the C entry point must reject the call with A1MPC_EINVAL after
ctypes has converted every argument against the declared prototype."""
import ctypes as C

import numpy as np
import pytest

from stance_scenarios import gains, robots


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_stance_binding_marshals_its_arguments(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    B = 4
    st = robots(B, 0)
    _, kdl, kpa, kda = gains("gazebo")
    args = [st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")] + [kdl, kpa, kda]
    for want_acc in (False, True):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            eng.stance_qp(*args, want_acc=want_acc)
    L = a1.lib()
    assert "a1mpc_stance_qp_batch" in a1.EXPORTS and hasattr(L, "a1mpc_stance_qp_batch")
    assert len(L.a1mpc_stance_qp_batch.argtypes) == 16
    assert L.a1mpc_stance_qp_batch(None, B, B, *([None] * 13)) == -1
    assert L.a1mpc_stance_qp_batch(None, B, C.c_size_t(2 ** 40), *([None] * 13)) == -1   # size_t ld is marshalled as such
    eng.h = None
