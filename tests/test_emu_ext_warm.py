"""The warm start of the scheduled call (a1mpc_solve_batch_ext_warm) on the lane-accurate CPU emulator, every QP against the
extended oracle.  Consecutive control ticks: the schedules are windows [t : t + 10] of one horizon-20 schedule (the generator
draws gait and phase before its step loop, so consecutive windows are consecutive ticks of the same gait, i.e. shift = 1), and
the state moves along the solver's own predicted trajectory for one step (plus a little noise), as a robot that follows its
plan does."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402

N = 10
WORDS = 4 + 4 * N
NOISE = np.array([.02, .02, .02, .01, .01, .005, .1, .1, .1, .05, .05, .05])[:, None]


@pytest.fixture(scope="module")
def E():
    import emu_py
    emu_py.lib()
    return emu_py


@pytest.fixture(scope="module")
def W(E):
    import emu_ext_warm_py
    emu_ext_warm_py.lib()
    return emu_ext_warm_py


@pytest.fixture(scope="module")
def a1(E):
    return E.a1mpc


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def advance(O, st, u, rng, noise):
    """one control tick: x1 = A_d x0 + B_d u0 of the condensed model (the first step of the plan), plus noise"""
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


def oracle(O, st, sched, normals):
    fo, info = O.compute_grf_batch_ext(O.make_config(horizon=N), obatch(O, st), sched, normals, mode=O.MODE_EXACT, nthreads=4)
    return fo


def _ticks(O, solve, st, s20, normals, T, warm, rng, noise=0.01):
    """T consecutive ticks through `solve`; per tick (f, status, iters, sched, oracle forces)"""
    out = []
    for t in range(T):
        sched = np.ascontiguousarray(s20[t:t + N])
        f, status, iters, u = solve(st, sched, warm)
        out.append((f, status, iters, sched, oracle(O, st, sched, normals)))
        st = advance(O, st, u, rng, noise)
    return out


@pytest.mark.parametrize("use_normals", [True, False])
def test_consecutive_ticks_general_kernel(W, a1, O, use_normals):
    B = 64
    cfg = a1.default_config(horizon=N)
    st = a1.gen_states(B, 4, 301)
    s20, normals = a1.gen_schedule(B, 20, 4, 301)
    nm = normals if use_normals else None
    s20[:, 0] = 0b1111                   # four feet down all the time
    s20[4, 1] = 0b0111                   # three feet in one step
    s20[:, 2] = 0b1001
    s20[10:, 2] |= 0b0010                # FR lands in the step that enters the horizon at tick 1, and stays
    s20[:, 3] = 0                        # no contact at all
    warm = np.full((B, WORDS), 0xFFFFFFFF, dtype=np.uint32)
    warm[:, 0] = 0                       # reset
    solve = lambda s, sc, w: W.solve(cfg, s, sc, nm, w, shift=1, want_u=True, order=2)
    ticks = _ticks(O, solve, st, s20, nm, 3, warm, np.random.default_rng(0))
    has = np.ones(B, dtype=bool); has[3] = False
    f0, s0, it0, _, fo0 = ticks[0]
    assert s0[3] == a1.STATUS_NO_CONTACT and (s0[has] == a1.STATUS_OPTIMAL).all() and np.abs(f0 - fo0).max() < 1e-7
    assert ((it0 % 100)[has] > 0).all()                  # empty slots: every robot took the cold path
    assert warm[3, 0] == 0 and (warm[has, 0] == 2).all()
    hits = []
    for f, status, iters, sched, fo in ticks[1:]:
        assert (status[has] == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7
        assert fact(iters)[has].mean() <= 0.5 * fact(it0)[has].mean(), (fact(iters)[has].mean(), fact(it0)[has].mean())
        hits.append(((iters % 100) == 0)[has].mean())
    assert min(hits) >= 0.8, hits                        # measured 0.84-0.95 (DESIGN 6c)


def test_consecutive_ticks_compact_kernel(W, a1, O):
    B = 64
    cfg = a1.default_config(horizon=N)
    st = a1.gen_states(B, 4, 302)
    s20, normals = a1.gen_schedule(B, 20, 4, 302)
    warm = np.zeros((B, WORDS), dtype=np.uint32)
    solve = lambda s, sc, w: W.solve_sched2(cfg, s, sc, normals, w, shift=1, want_u=True, order=1)
    ticks = _ticks(O, solve, st, s20, normals, 3, warm, np.random.default_rng(1))
    f0, s0, it0, _, fo0 = ticks[0]
    assert (s0 == a1.STATUS_OPTIMAL).all() and ((it0 % 100) > 0).all() and np.abs(f0 - fo0).max() < 1e-7
    for f, status, iters, sched, fo in ticks[1:]:
        assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7
        assert fact(iters).mean() <= 0.5 * fact(it0).mean()
        assert ((iters % 100) == 0).mean() >= 0.8


@pytest.mark.parametrize("first", ["general", "compact"])
def test_faces_carry_over_between_kernels(W, a1, O, first):
    """a robot may switch between the general and the compacted kernel from one tick to the next: the slot is per (step, leg)"""
    B = 48
    cfg = a1.default_config(horizon=N)
    st = a1.gen_states(B, 4, 303)
    s20, normals = a1.gen_schedule(B, 20, 4, 303)
    gen = lambda s, sc, w: W.solve(cfg, s, sc, normals, w, shift=1, want_u=True)
    cmp_ = lambda s, sc, w: W.solve_sched2(cfg, s, sc, normals, w, shift=1, want_u=True)
    order = (gen, cmp_) if first == "general" else (cmp_, gen)
    warm = np.zeros((B, WORDS), dtype=np.uint32)
    rng = np.random.default_rng(2)
    f, status, it0, u = order[0](st, np.ascontiguousarray(s20[0:N]), warm)
    assert (status == 0).all() and ((it0 % 100) > 0).all()
    st = advance(O, st, u, rng, 0.01)
    sched = np.ascontiguousarray(s20[1:N + 1])
    f, status, it1, u = order[1](st, sched, warm)
    assert (status == 0).all() and np.abs(f - oracle(O, st, sched, normals)).max() < 1e-7
    assert ((it1 % 100) == 0).mean() >= 0.8 and fact(it1).mean() <= 0.5 * fact(it0).mean()


def test_slot_kinds_and_garbage(E, W, a1, O):
    """a slot written by the constant-pattern warm call is "no guess" for the scheduled one and the reverse; a NaN robot stores no
    guess; a header with schedule bits past the horizon or impossible face codes is no guess"""
    B = 32
    cfg = a1.default_config(horizon=N)
    st = a1.gen_states(B, 2, 304)
    sched, normals = a1.gen_schedule(B, N, 4, 304)
    sched[:] = st["contact"][None, :]                    # the constant pattern, so that both calls pose the same QPs
    sched[:, st["contact"] == 0] = 0b0110
    st["contact"][:] = sched[0]
    cold = E.solve(cfg, st, sched=sched, normals=None)
    warm = np.zeros((B, WORDS), dtype=np.uint32)
    E.solve(cfg, st, warm=warm, shift=0)                  # constant-pattern slots (kind 1)
    assert (warm[:, 0] == 1).all()
    f, status, iters = W.solve(cfg, st, sched, None, warm, shift=0)
    assert (status == 0).all() and np.array_equal(iters, cold[2]) and np.abs(f - cold[0]).max() < 1e-12
    assert (warm[:, 0] == 2).all()
    f, status, iters, _ = E.solve(cfg, st, warm=warm, shift=0)   # and back: kind 2 is no guess for the constant-pattern call
    assert (status == 0).all() and ((iters % 100) > 0).all()
    # garbage: bits past the horizon, impossible face codes
    W.solve(cfg, st, sched, None, warm, shift=0)
    junk = warm.copy()
    junk[: B // 2, 3] |= 1 << 20
    junk[B // 2:, 4:] = 0xFFFFFFFF
    f, status, iters = W.solve(cfg, st, sched, None, junk, shift=0)
    assert (status == 0).all() and np.array_equal(iters, cold[2])
    # a NaN robot stores no guess, its neighbours do
    st["x0"][4, 5] = np.nan
    f, status, iters = W.solve(cfg, st, sched, normals, warm, shift=0)
    assert status[5] == a1.STATUS_NUMERICAL and np.abs(f[:, 5]).max() == 0 and warm[5, 0] == 0
    ok = np.arange(B) != 5
    assert (status[ok] == 0).all() and (warm[ok, 0] == 2).all()


def test_lane_order_does_not_matter(W, a1, O):
    B = 40
    cfg = a1.default_config(horizon=N)
    st = a1.gen_states(B, 4, 305)
    s20, normals = a1.gen_schedule(B, 20, 4, 305)
    s20[:, 0] = 0b1111
    s20[4, 1] = 0b0111
    w0 = np.zeros((B, WORDS), dtype=np.uint32)
    f, status, it, u = W.solve(cfg, st, np.ascontiguousarray(s20[:N]), normals, w0, shift=1, want_u=True)
    st = advance(O, st, u, np.random.default_rng(3), 0.01)
    sched = np.ascontiguousarray(s20[1:N + 1])
    res = []
    for order in (0, 1, 2):
        w = w0.copy()
        res.append(W.solve(cfg, st, sched, normals, w, shift=1, want_u=True, order=order) + (w,))
    for got in res[1:]:
        for a, b in zip(res[0], got):
            assert np.array_equal(a, b)
    assert ((res[0][2] % 100) == 0).mean() > 0.5
