"""CPU test of a1mpc_stance_qp_batch_ext, a1mpc_surface_normals_batch, a1mpc_tick_set_stance_terrain and their bindings: the prototypes in
include/a1mpc.h, the exports and ctypes argument types, and Engine.stance_qp_ext / Engine.surface_normals / Tick.set_stance_terrain
marshalling their arguments down to the C call, which rejects a NULL handle or tick with A1MPC_EINVAL before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("a1mpc_stance_qp_batch_ext", "a1mpc_surface_normals_batch", "a1mpc_tick_set_stance_terrain")


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def test_prototypes_and_exports(a1):
    hdr = open(os.path.join(ROOT, "include", "a1mpc.h")).read()
    assert re.search(r"int\s+a1mpc_stance_qp_batch_ext\(a1mpc_handle\* h, int B, size_t ld, const double\* x0, const double\* rot, "
                     r"const double\* rot_z, const double\* foot,\s+const uint32_t\* contact, const double\* des, const double\* kp_linear, "
                     r"const double\* kd_linear,\s+const double\* kp_angular, const double\* kd_angular, const double\* normals, double\* f_body, "
                     r"int32_t\* status,\s+double\* root_acc\);", hdr)
    assert re.search(r"int\s+a1mpc_surface_normals_batch\(a1mpc_handle\* h, int B, const void\* swing_state, const double\* root_pos, "
                     r"double\* normals\);", hdr)
    assert re.search(r"int\s+a1mpc_tick_set_stance_terrain\(a1mpc_tick\* t, int source, const double\* normals\);", hdr)
    for name in NAMES:
        assert name in a1.EXPORTS
    L = a1.lib()
    assert L.a1mpc_stance_qp_batch_ext.argtypes == [C.c_void_p, C.c_int, C.c_size_t] + [C.c_void_p] * 14
    assert L.a1mpc_surface_normals_batch.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    assert L.a1mpc_tick_set_stance_terrain.argtypes == [C.c_void_p, C.c_int, C.c_void_p]


def test_null_handle_and_tick_are_rejected(a1):
    L = a1.lib()
    B = 4
    buf = np.zeros((12, B))
    p = buf.ctypes.data
    assert L.a1mpc_stance_qp_batch_ext(None, B, B, *[p] * 14) == -1 and b"null argument" in L.a1mpc_last_error()
    assert L.a1mpc_surface_normals_batch(None, B, p, p, p) == -1 and b"null argument" in L.a1mpc_last_error()
    for source in (0, 1, 2, 7):
        assert L.a1mpc_tick_set_stance_terrain(None, source, p) == -1 and b"null argument" in L.a1mpc_last_error()


def _null_engine(a1):
    eng = a1.Engine.__new__(a1.Engine)
    eng.h, eng.cfg, eng.device = None, a1.default_config(), 0
    return eng


def test_bindings_marshal_their_arguments(a1):
    B = 4
    eng = _null_engine(a1)
    r = lambda rows: np.zeros((rows, B))
    with pytest.raises(a1.A1MpcError, match="null argument"):
        eng.stance_qp_ext(r(12), r(9), r(9), r(12), np.zeros(B), r(12), r(3), np.zeros(3), np.zeros(3), np.zeros(3), r(12), want_acc=True)
    with pytest.raises(a1.A1MpcError, match="null argument"):
        eng.surface_normals(None, r(3))
    tick = a1.Tick.__new__(a1.Tick)
    tick.eng, tick.B, tick.params, tick.t = eng, B, a1.default_tick_params(mode=a1.TICK_QP), None
    for source, ptr in ((a1.TERRAIN_FLAT, 0), (a1.TERRAIN_ESTIMATED, 0), (a1.TERRAIN_GIVEN, 0x1000), (a1.TERRAIN_GIVEN, None)):
        with pytest.raises(a1.A1MpcError, match="null argument"):
            tick.set_stance_terrain(source, ptr)
