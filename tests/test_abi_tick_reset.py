"""CPU test of a1mpc_tick_reset_robots and its bindings: the prototype in include/a1mpc.h, the ctypes argument types, Tick.reset_robots /
reset_robots_ptr marshalling their arguments down to the C call (which rejects the NULL tick with A1MPC_EINVAL), and the argument errors the
Python wrapper raises before any device work."""
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


def test_prototype_and_export(a1):
    hdr = open(os.path.join(ROOT, "include", "a1mpc.h")).read()
    assert re.search(r"int\s+a1mpc_tick_reset_robots\(a1mpc_tick\* t, const uint8_t\* mask\);", hdr)
    assert "a1mpc_tick_reset_robots" in a1.EXPORTS
    L = a1.lib()
    assert L.a1mpc_tick_reset_robots.argtypes == [C.c_void_p, C.c_void_p]


def test_null_tick_and_mask_are_rejected(a1):
    L = a1.lib()
    mask = np.ones(4, dtype=np.uint8)
    assert L.a1mpc_tick_reset_robots(None, mask.ctypes.data) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_tick_reset_robots(None, None) == -1 and b"null argument" in L.a1mpc_last_error()


def _null_tick(a1, B):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, a1.default_tick_params(), None
    return tick


def test_bindings_marshal_their_arguments(a1):
    B = 4
    tick = _null_tick(a1, B)
    # well-formed masks reach the C call, which rejects the NULL tick
    for mask in (np.zeros(B, dtype=bool), np.ones(B, dtype=np.uint8), np.array([True, False, True, False])[::1],
                 np.arange(2 * B, dtype=np.uint8)[::2]):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.reset_robots(mask)
    for ptr in (0x1000, None):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.reset_robots_ptr(ptr)


@pytest.mark.parametrize("bad", ["shape", "dtype", "2d"])
def test_reset_robots_rejects_malformed_masks(a1, bad):
    B = 4
    tick = _null_tick(a1, B)
    mask = dict(shape=np.ones(B + 1, dtype=bool), dtype=np.ones(B, dtype=np.int32), **{"2d": np.ones((1, B), dtype=bool)})[bad]
    with pytest.raises(ValueError, match="mask"):
        tick.reset_robots(mask)
