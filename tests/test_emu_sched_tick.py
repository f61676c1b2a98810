"""The scheduled MPC solve on the CPU emulator, on the QPs a closed-loop control tick poses (tests/sched_tick_scenarios.py: the
oracle chain's states, update_plan's schedules through standstill, walk / stand switches, early contacts and four-foot crossing
steps at all three gait speeds; variants plan, early and terrain).  Every QP of every tick against the extended oracle.

Cold: every QP through the general four-leg kernel (what A1MPC_EXT_COMPACT=0 does), and the QPs whose every step has two stance
feet also through the compacted kernel, so both halves of pack_ext2_kernel's routing are covered.  The emulator solves each QP on
its own, so the general kernel's result for a QP does not depend on which QPs share the call, and the cold solves of all ticks
go in one call.  Warm: the routed warm calls over consecutive ticks with shift = 1, one buffer per variant for the whole run,
through the toggles.

Checks: status OPTIMAL (NO_CONTACT exactly where the schedule has no contact), |f_body - f*| <= 1e-7 N and over the whole horizon
|u_full - u*| <= 1e-6 N.  A failure prints the failing QPs' inputs, schedule, tick and robot."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402
from sched_tick_scenarios import (VARIANTS, check_floors, describe, face_census, sched_census, stacked, tick_solve_inputs,  # noqa: E402
                                  two_feet, variant)

N = 10
WORDS = 4 + 4 * N
B, T, SEED = 16, 64, 41
TOL_F, TOL_U = 1e-7, 1e-6
# counts over the B x T = 1024 QPs of each variant.  Measured: 722 compacted / 302 general / 134 with a crossing step (plan);
# 545 / 479 / 293 and 18 with a three-foot step (early); oracle faces 966-972 QPs on a friction edge, 354-458 with a foot-step
# at the vertex, 66-187 with a whole foot at the vertex, 642-684 at fz_max
SCHED_FLOORS = {"plan": dict(compact=500, general=200, four=80, standstill=100, switch=16, early=150),
                "early": dict(compact=400, general=300, four=200, three=8, early=150),
                "terrain": dict(compact=500, general=200, four=80)}
FACE_FLOORS = {"plan": dict(edge=600, vertex=200, foot0=30, fzmax=300),
               "early": dict(edge=600, vertex=200, foot0=100, fzmax=300),
               "terrain": dict(edge=600, vertex=200, foot0=30, fzmax=300)}


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
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="module")
def D(O):
    """the run and the oracle's optimum (f, info, u_full) of every QP of every variant, stacked over the ticks; generated once"""
    d = tick_solve_inputs(B, T, SEED, N)
    ocfg = O.make_config(horizon=N)
    d["oracle"], d["stacked"] = {}, {}
    for name in VARIANTS:
        st, sched, normals = d["stacked"][name] = stacked(d, name)
        d["oracle"][name] = O.compute_grf_batch_ext(ocfg, obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
    return d


def check(a1, d, name, what, qps, f, status, u):
    """QPs `qps` (columns of stacked(d, name)) against the oracle; returns the largest errors in f and u"""
    sched = d["stacked"][name][1]
    fo, info, uo = d["oracle"][name]
    none = ~(sched[:, qps] != 0).any(axis=0)
    want = np.where(none, a1.STATUS_NO_CONTACT, a1.STATUS_OPTIMAL)
    ef = np.abs(f - fo[:, qps]).max(axis=0)
    eu = np.abs(u - uo[qps].T).max(axis=0)
    bad = np.nonzero((status != want) | ~(ef <= TOL_F) | ~(eu <= TOL_U) | ((info[qps, 1] != 1) & ~none))[0]
    assert bad.size == 0, "%s: %d QPs fail (status %s, |f - f*| %s, |u - u*| %s)\n%s" % (
        what, bad.size, status[bad][:8].tolist(), ef[bad][:8].tolist(), eu[bad][:8].tolist(), describe(d, name, qps[bad]))
    return np.array([ef.max(), eu.max()])


def _sub(st, sched, normals, sel):
    s = {k: np.ascontiguousarray(v[..., sel]) for k, v in st.items()}
    return s, np.ascontiguousarray(sched[:, sel]), (np.ascontiguousarray(normals[:, sel]) if normals is not None else None)


@pytest.mark.parametrize("name", VARIANTS)
def test_census(D, name):
    check_floors(name, sched_census(D, name), SCHED_FLOORS[name])
    check_floors(name + " faces", face_census(D, name, D["oracle"][name][2]), FACE_FLOORS[name])


@pytest.mark.parametrize("name", VARIANTS)
def test_cold_general_and_compacted(E, D, name):
    a1 = E.a1mpc
    cfg = a1.default_config(horizon=N)
    st, sched, normals = D["stacked"][name]
    every = np.arange(B * T)
    f, status, iters, u, _ = E.solve(cfg, st, sched=sched, normals=normals, want_u=True)
    worst = check(a1, D, name, "general kernel, " + name, every, f, status, u)
    two = np.nonzero(two_feet(sched))[0]
    s, sc, nm = _sub(st, sched, normals, two)
    f, status, iters, u = E.solve_sched2(cfg, s, sc, normals=nm, want_u=True)
    worst = np.maximum(worst, check(a1, D, name, "compacted kernel, " + name, two, f, status, u))
    print("%s cold: %d QPs on the general kernel, %d on the compacted kernel, max |f - f*| %.2e N, |u - u*| %.2e N" % (name, B * T, two.size, *worst))


def test_warm_routed_over_ticks(W, D):
    """per tick one call per kernel and normals kind: plan and early share the calls without normals (their buffers side by
    side), terrain has its own; each robot keeps its slot whichever kernel its schedule is routed to"""
    a1 = W.a1mpc
    cfg = a1.default_config(horizon=N)
    warm = {name: np.zeros((B, WORDS), dtype=np.uint32) for name in VARIANTS}
    worst = np.zeros(2)
    hits = {name: [] for name in VARIANTS}
    for t in range(T):
        for group in (("plan", "early"), ("terrain",)):
            st, sched, normals = stacked(D, group[0], [t])
            for name in group[1:]:
                s2, sc2, _ = variant(D, name, t)
                st = {k: np.concatenate([st[k], s2[k]], axis=-1) for k in st}
                sched = np.concatenate([sched, sc2], axis=1)
            w = np.concatenate([warm[name] for name in group])
            two = two_feet(sched)
            iters = np.zeros(w.shape[0], dtype=np.int64)
            for sel, solve, kernel in ((np.nonzero(two)[0], W.solve_sched2, "compacted"), (np.nonzero(~two)[0], W.solve, "general")):
                if sel.size == 0:
                    continue
                s, sc, nm = _sub(st, sched, normals, sel)
                ws = np.ascontiguousarray(w[sel])
                f, status, it, u = solve(cfg, s, sc, nm, ws, shift=1, want_u=True)
                w[sel] = ws
                iters[sel] = it
                for i, name in enumerate(group):
                    mine = (sel >= i * B) & (sel < (i + 1) * B)
                    qps = t * B + sel[mine] - i * B
                    worst = np.maximum(worst, check(a1, D, name, "warm %s kernel, %s tick %d" % (kernel, name, t), qps, f[:, mine], status[mine], u[:, mine]))
            for i, name in enumerate(group):
                warm[name] = w[i * B:(i + 1) * B]
                if t > 0:
                    hits[name].append(((iters[i * B:(i + 1) * B] % 100) == 0).mean())
    print("warm: max |f - f*| %.2e N, |u - u*| %.2e N; warm hits per tick, mean: %s" % (*worst, {k: round(float(np.mean(v)), 2) for k, v in hits.items()}))
    for name in VARIANTS:
        assert np.mean(hits[name]) > 0.3, (name, hits[name])   # measured 0.41-0.57: the loop exercises the warm path, not only its cold fall-back
