"""-m gpu: the warm start of the scheduled call (a1mpc_solve_batch_ext_warm) through the C ABI.  The closed loop is what the
call is for: a1mpc_update_plan_batch on device pointers produces each tick's schedule (one step further along the gait than the
last: shift = 1), the state follows the solver's own plan for one step, and every QP of every tick is checked against the
extended oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from common import obatch

pytestmark = pytest.mark.gpu

TOL_F = 1e-4
N = 10
NOISE = np.array([.02, .02, .02, .01, .01, .005, .1, .1, .1, .05, .05, .05])[:, None]


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def advance(O, st, u, rng, noise):
    ocfg = O.make_config(horizon=N)
    ob = obatch(O, st)
    st2 = {k: v.copy() for k, v in st.items()}
    for b in range(st["x0"].shape[1]):
        r = O.rollout(ocfg, ob, b)
        st2["x0"][:, b] = (r["A_d"] @ r["mpc_states"] + r["B_d_list"][:13] @ u[:12, b])[:12]
    st2["x0"] += noise * rng.standard_normal(st2["x0"].shape) * NOISE
    return st2


def fact(it):
    return it % 100 + it // 100


def _d2h(a1, eng, ptr, shape, dtype):
    x = np.zeros(shape, dtype=dtype)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, x.ctypes.data, ptr, x.nbytes))
    eng.sync()
    return x


def _h2d(a1, eng, ptr, x):
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, ptr, np.ascontiguousarray(x).ctypes.data, x.nbytes))


def test_closed_loop_with_update_plan(a1, O):
    B, T = 4096, 8
    eng = a1.Engine(a1.default_config(horizon=N))
    rng = np.random.default_rng(7)
    st = a1.gen_states(B, 4, 401)
    _, normals = a1.gen_schedule(B, N, 4, 401)
    gp = a1.default_gait_params(N)
    # trot, counters 12 per tick: a tenth of the gait over the horizon.  Phases on the 12-grid reach the counter boundary exactly
    # (a step with all four feet: general kernel); the others keep two feet per step (compacted kernel)
    phase = rng.integers(0, 20, B) * 12.0 + np.where(np.arange(B) % 2 == 0, 0.0, 5.0)
    gc = np.stack([phase, phase + 120.0, phase + 120.0, phase]) % 240.0
    d_gc = eng.dalloc(gc.nbytes); _h2d(a1, eng, d_gc, gc)
    d_sp = eng.dalloc(4 * B * 8); _h2d(a1, eng, d_sp, np.full((4, B), 12.0))
    d_mode = eng.dalloc(B * 4); _h2d(a1, eng, d_mode, np.ones(B, dtype=np.uint32))
    d_sched = eng.dalloc(N * B * 4)
    d_norm = eng.dalloc(12 * B * 8); _h2d(a1, eng, d_norm, normals)
    d = a1.DeviceBatch(eng, B, want_u=True)
    warm = eng.warm_alloc(B)
    ext = a1.InputsExt(d_sched.value, d_norm.value)
    ocfg = O.make_config(horizon=N)
    facts, both = [], False
    for t in range(T):
        a1._check(a1.lib().a1mpc_update_plan_batch(eng.h, B, C.byref(gp), d_gc, d_sp, d_mode, None, None, None, None, None, d.contact, d_sched,
                                                   None, None, None))
        d.upload({k: v for k, v in st.items() if k != "contact"} | {"contact": _d2h(a1, eng, d.contact, B, np.uint32)})
        a1._check(a1.lib().a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out), warm, 1))
        f, status = d.download()
        iters = _d2h(a1, eng, d.iters, B, np.int32)
        u = _d2h(a1, eng, d.u_full, (12 * N, B), np.float64)
        sched = _d2h(a1, eng, d_sched, (N, B), np.uint32)
        st["contact"] = sched[0].copy()
        fo, info = O.compute_grf_batch_ext(ocfg, obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
        assert (status == a1.STATUS_OPTIMAL).all(), (t, np.bincount(status))
        assert np.abs(f - fo).max() <= TOL_F, t
        two = np.array([bin(int(m)).count("1") == 2 for m in sched.reshape(-1)]).reshape(N, B).all(axis=0)
        both = both or (two.any() and (~two).any())
        facts.append(fact(iters).mean())
        if t == 0:
            assert ((iters % 100) > 0).all()
        st = advance(O, st, u, rng, 0.01)
    assert both
    assert max(facts[1:]) < 0.6 * facts[0], facts
    d.free()
    eng.close()


def test_first_call_matches_cold(a1):
    B = 2048
    eng = a1.Engine(a1.default_config(horizon=N))
    st = a1.gen_states(B, 4, 402)
    sched, normals = a1.gen_schedule(B, N, 4, 402)
    sched[:, 7] = 0b1111
    sched[:, 9] = 0
    warm = eng.warm_alloc(B)
    f, s, it = eng.solve_ext_warm(st, sched, normals, warm, shift=1)
    fc, sc, itc = eng.solve_ext(st, sched, normals)
    assert np.array_equal(s, sc) and s[9] == a1.STATUS_NO_CONTACT and (np.delete(s, 9) == 0).all()
    assert np.abs(f - fc).max() <= 1e-8
    # no schedule and no normals: a1mpc_solve_batch_warm
    f2, s2, it2 = eng.solve_ext_warm(st, None, None, warm, shift=0)
    fw, sw, itw = eng.solve(st)
    assert np.abs(f2 - fw).max() <= 1e-8
    eng.close()


def test_precision_32(a1, O):
    """fp32 boundary: |f - f*(fp32-rounded inputs)| <= 1e-4 N + 1 fp32 ulp (DESIGN 3), warm ticks included"""
    B = 1024
    eng = a1.Engine(a1.default_config(horizon=N, precision=32))
    st = a1.gen_states(B, 4, 403)
    s20, normals = a1.gen_schedule(B, 20, 4, 403)
    warm = eng.warm_alloc(B)
    rng = np.random.default_rng(4)
    its = []
    for t in range(3):
        sched = np.ascontiguousarray(s20[t:t + N])
        f, s, it, u = eng.solve_ext_warm(st, sched, normals, warm, shift=1, want_u=True)
        r = {k: (v if k == "contact" else v.astype(np.float32).astype(np.float64)) for k, v in st.items()}
        fo, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, r), sched, normals.astype(np.float32).astype(np.float64),
                                           O.MODE_EXACT, nthreads=O.hardware_threads())
        assert f.dtype == np.float32 and (s == 0).all()
        assert (np.abs(f - fo) <= TOL_F + np.abs(fo) * 2.0 ** -23).all()
        its.append(fact(it).mean())
        st = advance(O, st, u.astype(np.float64), rng, 0.01)
    assert its[2] < 0.6 * its[0], its
    eng.close()


def test_general_kernel_only(a1, O):
    """A1MPC_EXT_COMPACT=0 at a1mpc_create: every scheduled robot on the general kernel, warm start included"""
    os.environ["A1MPC_EXT_COMPACT"] = "0"
    try:
        eng = a1.Engine(a1.default_config(horizon=N))
    finally:
        del os.environ["A1MPC_EXT_COMPACT"]
    B = 1024
    st = a1.gen_states(B, 4, 404)
    s20, normals = a1.gen_schedule(B, 20, 4, 404)
    warm = eng.warm_alloc(B)
    rng = np.random.default_rng(5)
    its = []
    for t in range(3):
        sched = np.ascontiguousarray(s20[t:t + N])
        f, s, it, u = eng.solve_ext_warm(st, sched, normals, warm, shift=1, want_u=True)
        fo, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
        assert (s == 0).all() and np.abs(f - fo).max() <= TOL_F
        its.append(it)
        st = advance(O, st, u, rng, 0.01)
    assert ((its[0] % 100) > 0).all() and ((its[2] % 100) == 0).mean() > 0.75
    eng.close()


def test_argument_errors(a1):
    st = a1.gen_states(8, 4, 405)
    sched, normals = a1.gen_schedule(8, N, 4, 405)
    eng20 = a1.Engine(a1.default_config(horizon=20))
    s20, n20 = a1.gen_schedule(8, 20, 4, 405)
    w = eng20.dalloc(4096)
    with pytest.raises(a1.A1MpcError, match="horizon 10"):
        eng20.solve_ext_warm(st, s20, n20, w)
    eng20.close()
    eng = a1.Engine(a1.default_config(horizon=N))
    host = np.zeros(8 * 44, dtype=np.uint32)
    with pytest.raises(a1.A1MpcError, match="device memory"):
        eng.solve_ext_warm(st, sched, normals, host.ctypes.data_as(C.c_void_p))
    w = eng.warm_alloc(8)
    for shift in (-1, N + 1):
        with pytest.raises(a1.A1MpcError, match="shift out of range"):
            eng.solve_ext_warm(st, sched, normals, w, shift=shift)
    f, s, it = eng.solve_ext_warm(st, sched, normals, w, shift=N)
    assert (s == 0).all()
    eng.close()
