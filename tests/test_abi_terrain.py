"""CPU test of a1mpc_terrain_normals_batch, a1mpc_tick_set_terrain and their bindings: the prototypes and constants in include/a1mpc.h,
the ctypes argument types, and Engine.terrain_normals / Tick.set_terrain marshalling their arguments down to the C call, which rejects a
NULL handle or tick with A1MPC_EINVAL before any device work."""
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
    assert re.search(r"int\s+a1mpc_terrain_normals_batch\(a1mpc_handle\* h, int B, void\* swing_state, int use_terrain_adapt, const double\* root_pos, "
                     r"double\* ref,\s+size_t ref_ld, double\* terrain_pitch, double\* normals\);", hdr)
    assert re.search(r"int\s+a1mpc_tick_set_terrain\(a1mpc_tick\* t, int source, const double\* normals\);", hdr)
    consts = {k: int(v) for k, v in re.findall(r"#define (A1MPC_TERRAIN_\w+)\s+(\d+)", hdr)}
    assert consts == dict(A1MPC_TERRAIN_FLAT=0, A1MPC_TERRAIN_ESTIMATED=1, A1MPC_TERRAIN_GIVEN=2)
    assert (a1.TERRAIN_FLAT, a1.TERRAIN_ESTIMATED, a1.TERRAIN_GIVEN) == (0, 1, 2)
    for name in ("a1mpc_terrain_normals_batch", "a1mpc_tick_set_terrain"):
        assert name in a1.EXPORTS
    L = a1.lib()
    assert L.a1mpc_terrain_normals_batch.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                      C.c_void_p]
    assert L.a1mpc_tick_set_terrain.argtypes == [C.c_void_p, C.c_int, C.c_void_p]


def test_null_handle_and_tick_are_rejected(a1):
    L = a1.lib()
    B = 4
    buf = np.zeros((12, B))
    assert L.a1mpc_terrain_normals_batch(None, B, None, 1, None, None, B, None, None) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_terrain_normals_batch(None, B, buf.ctypes.data, 0, buf.ctypes.data, None, B, None, buf.ctypes.data) == -1
    for source in (0, 1, 2, 7):
        assert L.a1mpc_tick_set_terrain(None, source, buf.ctypes.data) == -1 and b"null argument" in L.a1mpc_last_error()


def _null_engine(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    return eng


def test_bindings_marshal_their_arguments(a1):
    B = 4
    eng = _null_engine(a1)
    r = lambda rows: np.zeros((rows, B))
    for call in (lambda: eng.terrain_normals(None, 1, r(3), r(9)), lambda: eng.terrain_normals(None, 0, r(3))):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            call()
    with pytest.raises(a1.A1MpcError, match="C-contiguous"):
        eng.terrain_normals(None, 1, r(3), np.zeros((B, 9)).T)
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, a1.default_tick_params(), None
    for source, ptr in ((a1.TERRAIN_FLAT, 0), (a1.TERRAIN_ESTIMATED, 0), (a1.TERRAIN_GIVEN, 0x1000), (a1.TERRAIN_GIVEN, None)):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.set_terrain(source, ptr)
