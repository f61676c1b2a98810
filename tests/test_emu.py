"""The device code of a1mpc_device.cuh on the lane-accurate CPU emulator (tests/emu/) against the oracle.

Test infrastructure, not a product path: the SAME kernels nvcc compiles for sm_90a are compiled by g++ against an
emulation of the warp primitives (shuffles, ballots, mma.m8n8k4.f64 fragments, __syncwarp) and run one fibre per CUDA
thread.  This catches, without a GPU, what the oracle alone cannot: wrong fragment/lane maps, wrong shared-memory tile
addressing, missing barriers (results must not depend on the order in which the lanes of a warp run between two
collectives), misaligned 128-bit shared accesses.  The GPU parity tests (-m gpu) remain the gate for the real thing."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402

TOL_F = 1e-4   # N, the gate of the GPU parity tests (SURVEY 8c P1)


@pytest.fixture(scope="module")
def E():
    import emu_py
    emu_py.lib()
    return emu_py


@pytest.fixture(scope="module")
def a1(E):
    return E.a1mpc


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _mixed_states(a1, B, config_id, stream):
    st = a1.gen_states(B, config_id, stream)
    pats = [1, 2, 4, 8, 3, 5, 6, 9, 10, 12, 7, 11, 13, 14, 15, 0]
    for i in range(min(B, len(pats))):
        st["contact"][i] = pats[i]
    return st


@pytest.mark.parametrize("horizon,B", [(10, 96), (20, 24)])
def test_fused_kernels_on_emulator_match_oracle(E, a1, O, horizon, B):
    cfg = a1.default_config(horizon=horizon)
    st = _mixed_states(a1, B, 2, 17)
    f, status, iters, u, stats = E.solve(cfg, st, order=0, want_u=True)
    assert stats["collectives"] > 0
    fo, info, uo = O.compute_grf_batch(O.make_config(horizon=horizon), obatch(O, st), mode=O.MODE_EXACT, nthreads=4, want_u=True)
    nc = st["contact"] == 0
    assert (status[nc] == a1.STATUS_NO_CONTACT).all() and (status[~nc] == a1.STATUS_OPTIMAL).all()
    assert np.abs(f - fo).max() <= TOL_F and np.abs(f - fo).max() < 1e-6
    assert np.abs(u - uo.T).max() <= TOL_F


def test_lane_order_between_collectives_does_not_matter(E, a1):
    """a missing __syncwarp around shared memory shows up as an order-dependent result"""
    cfg = a1.default_config(horizon=10)
    st = _mixed_states(a1, 48, 2, 23)
    ref = E.solve(cfg, st, order=0, want_u=True)
    for order in (1, 2):
        got = E.solve(cfg, st, order=order, want_u=True)
        assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1]) and np.array_equal(ref[2], got[2])
        assert np.array_equal(ref[3], got[3])


@pytest.mark.parametrize("horizon,B", [(10, 96), (20, 16)])
def test_config4_schedules_and_normals_on_emulator(E, a1, O, horizon, B):
    """shared memory is poisoned with NaN in the emulator: a never-written word that reaches a result fails this test (the
    barrier slots of absent foot-steps did, before they were masked)"""
    st = a1.gen_states(B, 4, 131)
    sched, normals = a1.gen_schedule(B, horizon, 4, 131)
    sched[:, 0] = 0                      # no contact anywhere in the horizon
    sched[:, 1] = 0b1111                 # all four feet all the time, tilted terrain only
    sched[1:, 2] = 0                     # contact in the first step only
    sched[0, 3] = 0                      # nobody in contact in the step whose force is returned
    cfg = a1.default_config(horizon=horizon)
    f, status, iters, stats = E.solve(cfg, st, sched=sched, normals=normals, order=2)
    fo, info = O.compute_grf_batch_ext(O.make_config(horizon=horizon), obatch(O, st), sched, normals, mode=O.MODE_EXACT, nthreads=4)
    assert status[0] == a1.STATUS_NO_CONTACT and (status[1:] == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= TOL_F


@pytest.mark.parametrize("horizon", [10, 20])      # 20: the direct classes run as a team of warps (Geo::TW)
def test_dense_solve_on_emulator(E, a1, O, horizon):
    B = 10
    st = a1.gen_states(B, 4, 91)
    st["contact"][:6] = [0b0001, 0b0111, 0b1111, 0b0110, 0b1000, 0]
    cfg = a1.default_config(horizon=horizon)
    ocfg = O.make_config(horizon=horizon)
    ob = obatch(O, st)
    Hg = [O.build_qp(ocfg, ob, b) for b in range(B)]
    H = np.stack([x[0] for x in Hg]); g = np.stack([x[1] for x in Hg])
    u, status = E.solve_dense(cfg, H, g, st["contact"], order=1)
    for b in range(B):
        if st["contact"][b] == 0:
            assert status[b] == a1.STATUS_NO_CONTACT and np.abs(u[b]).max() == 0
            continue
        if horizon == 20 and bin(int(st["contact"][b])).count("1") >= 3:
            continue       # the library reports these as unsupported at N = 20 (dense H + factor exceed shared memory); not emulated
        uo, info = O.solve_dense(ocfg, H[b], g[b], st["contact"][b], O.MODE_EXACT)
        assert status[b] == 0 and np.abs(u[b] - uo).max() <= TOL_F, (b, status[b])


def test_grf_qp_on_emulator(E, a1, O):
    rng = np.random.default_rng(5)
    B = 24
    st = a1.gen_states(B, 2, 101)
    rot = st["rot"].T.copy()
    yaw = st["x0"][2]
    rot_z = np.stack([np.cos(yaw), -np.sin(yaw), 0 * yaw, np.sin(yaw), np.cos(yaw), 0 * yaw, 0 * yaw, 0 * yaw, 1 + 0 * yaw], axis=1)
    foot = st["foot"].T.copy()
    acc = np.stack([rng.normal(0, 20, B), rng.normal(0, 20, B), 12 * 9.8 + rng.normal(0, 30, B), rng.normal(0, 5, B), rng.normal(0, 5, B),
                    rng.normal(0, 2, B)], axis=1)
    contact = st["contact"].copy()
    contact[:6] = [0b1111, 0b0001, 0b0111, 0, 0b1010, 0b1111]
    acc[5] = [400, -300, 2500, 50, -40, 10]
    f, status = E.grf_qp(acc, rot_z, rot, foot, contact, order=2)
    for b in range(B):
        if contact[b] == 0:
            assert status[b] == a1.STATUS_NO_CONTACT and np.abs(f[b]).max() == 0
            continue
        fo, info = O.grf_qp_single(acc[b], rot_z[b], rot[b], foot[b], contact[b], O.MODE_EXACT)
        assert status[b] == 0 and np.abs(f[b] - fo).max() <= TOL_F, (b, status[b])


def test_degenerate_vertex_family_is_certified(E, a1, O):
    """The one QP of the 1.44 M robustness sweep on the GPU that ended IPM_ONLY, with
    1e-9 perturbations: at one foot-step the optimum is the cone vertex with a degenerate multiplier; release (dual violation
    4e-11, just above the 1e-11 certificate tolerance) and re-pin (fz = -2.6e-7) alternated for all 36 rounds.  Without the
    residual-driven refinement of the reduced solves (variant "nohyst": fixed step count as in round 1, no hysteresis either) the
    status says so -- never a silent wrong answer; with it (the default) the false violation is gone and every copy is certified."""
    d = dict(np.load(os.path.join(ROOT, "tools", "data", "hard_qp_63168.npz")))
    n = 96
    rng = np.random.default_rng(3)
    st = {k: (np.repeat(v[:1], n) if k == "contact" else np.repeat(v[:, :1], n, axis=1).copy()) for k, v in d.items()}
    st["x0"] += 1e-9 * rng.standard_normal(st["x0"].shape)
    cfg = a1.default_config(horizon=10)
    fo, info = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, st), mode=O.MODE_EXACT, nthreads=4)
    f, status, iters, _ = E.solve(cfg, st)
    assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7 and (iters // 100).max() <= 6
    f0, status0, iters0, _ = E.solve(cfg, st, variant="nohyst")
    assert set(np.unique(status0)) == {a1.STATUS_OPTIMAL, a1.STATUS_IPM_ONLY}            # the cycle, reported as such
    assert np.abs(f0 - fo)[:, status0 == a1.STATUS_OPTIMAL].max() < 1e-7 and np.abs(f0 - fo).max() < 1e-2


def test_false_dual_violation_from_an_under_refined_solve(E, a1, O):
    """QP 618 of an emulator sweep (config 4, seed 777, three stance feet): the wrench-space reduced system of the finisher,
    refined once, left 1e-7 of residual on a free coordinate; that showed up as a dual violation of 4e-7 at a foot-step whose
    optimum IS the cone vertex -- release, primal violation (fz = -2e-4), re-pin, for all 36 rounds, status IPM_ONLY and 2e-3 N
    off.  With the reduced solves refined until the stationarity residual is <= 1e-11: verified in round 3."""
    d = dict(np.load(os.path.join(ROOT, "tools", "data", "hard_qp_777_618.npz")))
    cfg = a1.default_config(horizon=10)
    fo, info = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, d), mode=O.MODE_EXACT, nthreads=1)
    f, status, iters, _ = E.solve(cfg, d)
    assert status[0] == a1.STATUS_OPTIMAL and np.abs(f - fo).max() < 1e-7 and iters[0] // 100 <= 6
    f0, status0, iters0, _ = E.solve(cfg, d, variant="nohyst")
    assert status0[0] == a1.STATUS_IPM_ONLY and iters0[0] // 100 == 36 and 1e-4 < np.abs(f0 - fo).max() < 1e-2


def test_warm_start_across_ticks_on_emulator(E, a1, O):
    """SURVEY 8f.3: the device-resident warm start (a1mpc_solve_batch_warm) -- the previous tick's verified active faces are the
    first guess of the finisher; a hit costs 1-2 reduced factorisations and no interior-point iteration, a miss falls back to
    the cold path; the optimum is the same either way."""
    B = 160
    cfg = a1.default_config(horizon=10)
    st = a1.gen_states(B, 2, 5)
    for i, p in enumerate([1, 2, 4, 8, 7, 11, 13, 14, 15, 0]):
        st["contact"][i] = p
    warm = np.zeros((B, 4 + 4 * 10), dtype=np.uint32)
    f1, s1, it1, _ = E.solve(cfg, st, warm=warm, shift=0)
    nz = st["contact"] != 0
    assert (s1[nz] == a1.STATUS_OPTIMAL).all() and (warm[nz, 0] == 1).all() and (warm[~nz, 0] == 0).all()
    assert ((it1 % 100)[nz] > 0).all()                       # no guess yet: every robot took the interior-point path
    fo1, _ = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, st), mode=O.MODE_EXACT, nthreads=4)
    assert np.abs(f1 - fo1).max() <= TOL_F
    # next tick: the state advances by dt plus sensor-level noise; a few robots change their stance set
    rng = np.random.default_rng(0)
    st2 = {k: v.copy() for k, v in st.items()}
    st2["x0"][3:6] += 0.0025 * st["x0"][9:12]
    st2["x0"][0:3] += 0.0025 * st["x0"][6:9]
    st2["x0"] += 0.03 * rng.standard_normal(st2["x0"].shape) * np.array([.02, .02, .02, .01, .01, .005, .1, .1, .1, .05, .05, .05])[:, None]
    st2["contact"][20:24] = [3, 5, 15, 6]
    changed = st2["contact"] != st["contact"]
    f2, s2, it2, _ = E.solve(cfg, st2, warm=warm, shift=0, order=2)
    fo2, _ = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, st2), mode=O.MODE_EXACT, nthreads=4)
    assert (s2[nz] == a1.STATUS_OPTIMAL).all() and np.abs(f2 - fo2).max() <= TOL_F and np.abs(f2 - fo2).max() < 1e-7
    hit = ((it2 % 100) == 0) & nz
    assert not hit[changed].any()                            # different stance feet: cold start
    assert hit[nz & ~changed].mean() > 0.8                   # most robots keep their active faces from one tick to the next
    fact_warm = (it2 % 100 + it2 // 100)[nz & ~changed].mean()
    fact_cold = (it1 % 100 + it1 // 100)[nz].mean()
    assert fact_warm < 0.5 * fact_cold, (fact_warm, fact_cold)


def test_leg_kinematics_and_ekf_on_emulator(E, O):
    """SURVEY 8f.4 on the emulator: the batched FK/Jacobian kernel against the (reference-pinned) oracle, and 20 ticks of the
    batched Kalman filter (DMMA Cholesky of the 28x28 innovation covariance, eight right-hand sides per solve) next to the
    oracle's dense restatement, each carrying its own state"""
    from common import check_kinematics, ekf_walk, estimation_scenario
    rng, rho_opt, rho_fix, q, dq, rot = estimation_scenario(48, 1)
    check_kinematics(O, E.leg_kinematics(q, dq, rot, rho_opt.reshape(12), rho_fix.reshape(20)), q, dq, rot, rho_opt, rho_fix)
    box = {}

    def init(fpr, rot_):
        box["s"] = E.ekf_init(fpr, rot_)
        return lambda: (box["s"][:, :18], box["s"][:, 18:].reshape(-1, 18, 18))

    def update(dt, flat, mode, acc, gyro, rot_, fpr, fvr, force, tick):
        return E.ekf_update(box["s"], dt, flat, mode, acc, gyro, rot_, fpr, fvr, force, order=tick % 3)
    worst = ekf_walk(O, 40, 20, E.leg_kinematics, init, update, seed=2)
    assert worst < 1e-11, worst


def test_compact_two_feet_schedule_kernel_on_emulator(E, a1, O):
    """a1mpc_sched.cuh: config-4 schedules with two stance feet per step as a 60-variable direct problem (legs change from step
    to step; full 12x12 Gram blocks + (step, leg) selection), with and without terrain normals, against the extended oracle"""
    B = 120
    st = a1.gen_states(B, 4, 55)
    sched, normals = a1.gen_schedule(B, 10, 4, 55)
    assert all(bin(int(m) & 15).count("1") == 2 for m in sched.reshape(-1))      # trot / bound / gallop phases of the generator
    cfg = a1.default_config(horizon=10)
    for nm in (normals, None):
        f, status, iters, u = E.solve_sched2(cfg, st, sched, nm, order=2, want_u=True)
        fo, info, uo = O.compute_grf_batch_ext(O.make_config(horizon=10), obatch(O, st), sched, nm, mode=O.MODE_EXACT, nthreads=4, want_u=True)
        assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7 and np.abs(u.T - uo).max() < 1e-7


def test_edge_cases_on_emulator(E, a1, O):
    """NaN / Inf inputs, no stance foot, bits above the four legs -- statuses and zero forces, neighbours unaffected; the same through
    the warm-start kernels (a robot that was NUMERICAL stores no guess)"""
    st = a1.gen_states(40, 2, 51)
    st["contact"][0] = 0
    st["contact"][1] = 0b10000
    st["x0"][5, 2] = np.nan
    st["foot"][3, 3] = np.inf
    cfg = a1.default_config(horizon=10)
    warm = np.zeros((40, 44), dtype=np.uint32)
    for kw in ({}, {"warm": warm, "shift": 0}):
        f, status, iters, _ = E.solve(cfg, st, **kw)
        assert status[0] == a1.STATUS_NO_CONTACT and status[1] == a1.STATUS_NO_CONTACT and np.abs(f[:, :2]).max() == 0
        assert status[2] == a1.STATUS_NUMERICAL and status[3] == a1.STATUS_NUMERICAL and np.abs(f[:, 2:4]).max() == 0
        ok = np.arange(40) >= 4
        fo, info = O.compute_grf_batch(O.make_config(), obatch(O, st, slice(4, 40)), O.MODE_EXACT, nthreads=4)
        assert (status[ok] == 0).all() and np.abs(f[:, ok] - fo).max() <= TOL_F
    assert (warm[2:4, 0] == 0).all() and (warm[4:, 0] == 1).all()


def test_certified_means_optimal_every_qp_checked(E, a1, O):
    """OPTIMAL must mean optimal.  (1) The QPs that round 1's certificate got wrong -- stationarity on the free coordinates was
    assumed after the linear solve; three stance feet, Woodbury residual 3e-4, certified 1.8e-2 N / 5.9e-4 N off -- and the two
    warm-started ones that the finisher hysteresis certified 2e-4 N / 1.7e-5 N off.  (2) Every QP of a
    batch with random stance patterns against the oracle, not a sample."""
    cfg = a1.default_config(horizon=10)
    d = dict(np.load(os.path.join(ROOT, "tools", "data", "false_certificates_r01.npz")))
    fo, info = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, d), mode=O.MODE_EXACT, nthreads=2)
    f, status, iters, _ = E.solve(cfg, d)
    assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7
    f0, status0, _, _ = E.solve(cfg, d, variant="nohyst")                 # round-1 certificate: OPTIMAL and wrong
    assert (status0 == a1.STATUS_OPTIMAL).all() and np.abs(f0 - fo).max() > 1e-4
    w = dict(np.load(os.path.join(ROOT, "tools", "data", "false_certificates_warm_r01.npz")))
    warm = np.ascontiguousarray(w.pop("warm"))
    fo, info = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, w), mode=O.MODE_EXACT, nthreads=2)
    f, status, iters, _ = E.solve(cfg, w, warm=warm, shift=0)
    assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7
    B = 1500
    st = a1.gen_states(B, 4, 2024)
    st["contact"][:] = np.random.default_rng(5).integers(1, 16, size=B).astype(np.uint32)
    fo, info = O.compute_grf_batch(O.make_config(horizon=10), obatch(O, st), mode=O.MODE_EXACT, nthreads=4)
    f, status, iters, _ = E.solve(cfg, st)
    assert (info[:, 1] == 1).all() and (status == a1.STATUS_OPTIMAL).all()
    assert np.abs(f - fo).max() < 1e-7, np.abs(f - fo).max()
