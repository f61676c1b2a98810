"""a1mpc_solve_dense_batch on the CPU emulator of the device code, on QPs with a different B_d per horizon step (tests/dense_scenarios.py):
the route of a caller that builds H, g with ConvexMpc::calculate_qp_mats from its own B_mat_d_list (a1mpc_qp_mats_batch, then this
solve).  dense_solve_kernel<NS,N> runs nowhere else: the direct 90 x 90 and 120 x 120 factors of three and four stance feet at N = 10,
and the two-warp team of one and two feet at N = 20.

- every QP of four families (256 per family at N = 10, every stance class; 64 at N = 20, one or two feet) against the oracle's exact
  solve of the same H, g, to 1e-7 N over the whole horizon, with floors on the census of the oracle's optimum and on how much B_d
  moves from step to step;
- a class with more QPs than blocks: the grid capped at 1-3 blocks, under each lane order, gives the bits of one block per QP, on a
  batch where QPs that end NUMERICAL or have no stance foot sit between good ones, so a block solves a good QP right after a bad one;
- the input contract: the strict lower triangle and the swing rows and columns are never read; a non-finite or huge stance entry
  anywhere in the upper triangle, a non-positive stance diagonal or a non-finite gradient gives NUMERICAL with u all zero;
- at N = 20 the three- and four-foot classes are reported NUMERICAL with u all zero;
- compute_grf's 12-variable QP (a1mpc_grf_qp_batch, the other dense_solve-style loop of a1mpc_dense.cu) gives the same bits with its grid
  capped.

tests/emu/emu_dense.cpp launches these kernels as a1mpc_dense.cu's host code does, with a grid cap per class."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import dense_scenarios as DS  # noqa: E402
from common import obatch  # noqa: E402
from envelope_scenarios import census, check_census  # noqa: E402

TOL_CERT = 1e-7     # N, over the whole horizon
SEED = 97
SIZES = {10: (256, (1, 2, 3, 4)), 20: (64, (1, 2))}


@pytest.fixture(scope="module")
def E():
    import emu_dense_py
    emu_dense_py.lib()
    return emu_dense_py


@pytest.fixture(scope="module")
def a1(E):
    return E.a1mpc


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


def _cores():
    return max(1, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1))


def _family(a1, O, name, horizon, B=None, counts=None):
    b0, c0 = SIZES[horizon]
    ocfg = O.make_config(horizon=horizon)
    d = DS.build(a1, ocfg, name, B or b0, SEED, counts or c0)
    H, g = DS.qp_mats(O, ocfg, d, range(len(d["contact"])))
    return d, H, g


@pytest.mark.parametrize("horizon", [10, 20])
def test_per_step_model_is_the_oracle_rollout(a1, O, horizon):
    """the numpy B_d of step k is the oracle's B_d of the state posed at step k; A_d, x0, x_d are the rollout's; with B_d held constant
    calculate_qp_mats gives build_qp's H, g"""
    ocfg = O.make_config(horizon=horizon)
    for name in DS.FAMILIES:
        d = DS.build(a1, ocfg, name, 16, SEED, SIZES[horizon][1])
        assert DS.pin_rollout(O, ocfg, d, range(0, 16, 5)) <= 1e-13, name
        st = d["st"]
        for b in range(0, 16, 5):
            Hc, gc = O.qp_mats(ocfg, d["A_d"][b], d["B_const"][b], d["x0"][b], d["x_d"][b])
            Hb, gb, _, _, _ = O.build_qp(ocfg, obatch(O, st), b)
            assert np.abs(Hc - Hb).max() <= 1e-13 * np.abs(Hb).max() and np.abs(gc - gb).max() <= 1e-12 * np.abs(gb).max(), (name, b)


@pytest.mark.parametrize("name", DS.FAMILIES)
@pytest.mark.parametrize("horizon", [10, 20])
def test_every_per_step_qp_matches_the_oracle(E, a1, O, horizon, name):
    d, H, g = _family(a1, O, name, horizon)
    ocfg = O.make_config(horizon=horizon)
    contact = d["contact"]
    uo, cert = DS.oracle_solve(O, ocfg, H, g, contact, nthreads=_cores())
    assert cert.all()
    check_census("%s N=%d" % (name, horizon), census(uo, contact), DS.CENSUS_FLOORS[horizon])
    DS.check_bd_step(name, d)
    u, status = E.solve_dense(a1.default_config(horizon=horizon), H, g, contact, order=2, nthreads=_cores())
    err = np.abs(u - uo).max(axis=1)
    ns = np.array([bin(int(c)).count("1") for c in contact])
    print("%-9s N=%d worst |u - u*| per stance count: %s" % (name, horizon, "  ".join("%d: %.1e (%d QPs)" % (k, err[ns == k].max(), (ns == k).sum())
                                                                                        for k in range(1, 5) if (ns == k).any())))
    assert (status == a1.STATUS_OPTIMAL).all(), (np.bincount(status), np.nonzero(status)[0][:10])
    assert err.max() <= TOL_CERT, (err.max(), int(err.argmax()), int(contact[err.argmax()]))


def _contract(a1, O, horizon, B):
    """a small clean batch of the combined family (every class of the horizon) and the contract cases applied to it"""
    d, H, g = _family(a1, O, "combined", horizon, B=B)
    return (H, g, d["contact"]) + DS.contract_batch(H, g, d["contact"], horizon)


@pytest.mark.parametrize("horizon,B", [(10, 48), (20, 40)])
def test_input_contract(E, a1, O, horizon, B):
    H, g, contact, Hx, gx, cx, labels = _contract(a1, O, horizon, B)
    cfg = a1.default_config(horizon=horizon)
    u0, s0 = E.solve_dense(cfg, H, g, contact, nthreads=_cores())
    assert (s0 == a1.STATUS_OPTIMAL).all()
    u, status = E.solve_dense(cfg, Hx, gx, cx, order=1, nthreads=_cores())
    DS.check_contract(a1, u, status, u0, s0, labels)


@pytest.mark.parametrize("horizon,B", [(10, 48), (20, 40)])
def test_blocks_that_loop_over_their_class_give_the_same_bits(E, a1, O, horizon, B):
    """a block that solves several QPs in turn reuses its shared memory (the Hessian, the factor, the face state, the padding that
    only the team's warp 0 writes); nothing of one QP may reach the next"""
    _, _, _, Hx, gx, cx, labels = _contract(a1, O, horizon, B)
    cfg = a1.default_config(horizon=horizon)
    ref = E.solve_dense(cfg, Hx, gx, cx, order=0, nthreads=_cores())
    assert {int(s) for s in ref[1]} == {a1.STATUS_OPTIMAL, a1.STATUS_NUMERICAL, a1.STATUS_NO_CONTACT}
    for cap in (1, 2, 3):
        for order in (0, 1, 2):
            u, status = E.solve_dense(cfg, Hx, gx, cx, order=order, max_blocks=cap, nthreads=_cores())
            assert np.array_equal(status, ref[1]) and np.array_equal(u, ref[0]), (cap, order)


def test_n20_three_and_four_feet_are_reported_unsupported(E, a1, O):
    """the 180 x 180 and 240 x 240 direct factors do not fit in shared memory: those QPs end NUMERICAL with u written as zeros, and the
    one- and two-foot QPs of the same batch are solved as if alone"""
    d_bad, H_bad, g_bad = _family(a1, O, "push", 20, B=12, counts=(3, 4))
    d_ok, H_ok, g_ok = _family(a1, O, "push", 20, B=12, counts=(1, 2))
    H = np.concatenate([H_bad, H_ok]); g = np.concatenate([g_bad, g_ok]); contact = np.concatenate([d_bad["contact"], d_ok["contact"]])
    perm = np.random.default_rng(1).permutation(len(contact))
    cfg = a1.default_config(horizon=20)
    u, status = E.solve_dense(cfg, H[perm], g[perm], contact[perm], nthreads=_cores())
    bad = perm < 12
    assert (status[bad] == a1.STATUS_NUMERICAL).all() and np.array_equal(u[bad], np.zeros_like(u[bad])), status[bad]
    u1, s1 = E.solve_dense(cfg, H_ok, g_ok, d_ok["contact"], nthreads=_cores())
    assert (s1 == a1.STATUS_OPTIMAL).all()
    assert np.array_equal(status[~bad], s1[perm[~bad] - 12]) and np.array_equal(u[~bad], u1[perm[~bad] - 12])


def test_grf_qp_blocks_that_loop_over_their_class_give_the_same_bits(E, a1, O):
    """grf_qp_kernel<NS> loops over its class as dense_solve_kernel does; a block that solves a saturated or no-contact QP and then a
    good one gives the bits of one block per QP, and the QPs match the oracle"""
    rng = np.random.default_rng(5)
    B = 48
    st = a1.gen_states(B, 2, 101)
    rot = st["rot"].T.copy()
    yaw = st["x0"][2]
    rot_z = np.stack([np.cos(yaw), -np.sin(yaw), 0 * yaw, np.sin(yaw), np.cos(yaw), 0 * yaw, 0 * yaw, 0 * yaw, 1 + 0 * yaw], axis=1)
    foot = st["foot"].T.copy()
    acc = np.stack([rng.normal(0, 20, B), rng.normal(0, 20, B), 12 * 9.8 + rng.normal(0, 30, B), rng.normal(0, 5, B), rng.normal(0, 5, B),
                    rng.normal(0, 2, B)], axis=1)
    contact = DS.draw_contact(rng, B, (1, 2, 3, 4))
    contact[::7] = 0
    acc[3::5] = [400, -300, 2500, 50, -40, 10]          # fz_max and the friction faces
    acc[4] = np.nan                                     # non-finite wrench: NUMERICAL, zero forces
    ref = E.grf_qp(acc, rot_z, rot, foot, contact, order=0)
    assert ref[1][4] == a1.STATUS_NUMERICAL and np.abs(ref[0][4]).max() == 0
    for b in range(B):
        if b == 4:
            continue
        if contact[b] == 0:
            assert ref[1][b] == a1.STATUS_NO_CONTACT and np.abs(ref[0][b]).max() == 0
            continue
        fo, info = O.grf_qp_single(acc[b], rot_z[b], rot[b], foot[b], contact[b], O.MODE_EXACT)
        assert ref[1][b] == a1.STATUS_OPTIMAL and np.abs(ref[0][b] - fo).max() <= TOL_CERT, (b, ref[1][b])
    for cap in (1, 2, 3):
        for order in (0, 1, 2):
            f, status = E.grf_qp(acc, rot_z, rot, foot, contact, order=order, max_blocks=cap)
            assert np.array_equal(status, ref[1]) and np.array_equal(f, ref[0]), (cap, order)
