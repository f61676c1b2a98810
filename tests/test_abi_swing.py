"""CPU test of the bindings of the swing-leg / terrain entry points: with a NULL handle every C entry point must reject the call with
A1MPC_EINVAL after ctypes has converted every argument against the declared prototype."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_swing_bindings_marshal_their_arguments(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    B = 4
    null = C.c_void_p(0)
    rng = np.random.default_rng(0)
    r = lambda *s: rng.standard_normal(s)
    gp = a1.default_gait_params(10)
    calls = [
        lambda: eng.swing_alloc(B),
        lambda: eng.swing_init(null, B),
        lambda: eng.swing_legs(gp, r(12), r(12), null, 0.0025, r(4, B), np.ones(B, dtype=np.uint32), r(9, B), r(12, B), r(12, B), r(4, B)),
        lambda: eng.terrain_pitch(null, 1, r(3, B), np.zeros((9, B))),
        lambda: eng.terrain_pitch(null, 0, r(3, B)),
    ]
    for call in calls:
        with pytest.raises(a1.A1MpcError, match="null argument"):
            call()
    L = a1.lib()
    assert L.a1mpc_swing_bytes(B) == B * 921 * 8 and L.a1mpc_swing_bytes(0) == 0
    assert L.a1mpc_swing_init_batch(None, B, None) == -1
    assert L.a1mpc_terrain_pitch_batch(None, B, None, 1, None, None, B, None) == -1
    eng.h = None
