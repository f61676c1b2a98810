"""-m gpu: a1mpc_solve_dense_batch on QPs with a different B_d per horizon step (tests/dense_scenarios.py), the route of a caller that
gives ConvexMpc::calculate_qp_mats its own B_mat_d_list: a1mpc_qp_mats_batch into a1mpc_solve_dense_batch on device arrays.

- the chain at B = 8192 (N = 10, every stance class) and B = 2048 (N = 20, one or two feet) per family, so every class's CTAs solve
  several QPs in turn: every QP OPTIMAL; on a seeded subset of 512 QPs per family, H and g within the P0 tolerances of the oracle's
  calculate_qp_mats and u within 1e-7 N of the oracle's exact solve;
- the same states with a constant B_d: the dense solve of build_qp's H, g against the fused solve's whole-horizon u (the Kronecker or
  wrench-space form of the same QP) to 2e-7 N, both OPTIMAL, on every QP;
- a permuted batch (other CTAs, other order) and a repeated run give the same bits;
- the input contract among 8192 clean QPs, whose results must not move: the strict lower triangle and the swing rows and columns are
  never read; NaN, Inf or 1e300 anywhere in the stance upper triangle, a non-positive stance diagonal or a non-finite gradient give
  NUMERICAL with u all zero; no stance foot gives NO_CONTACT; at N = 20 three or four feet give NUMERICAL with u all zero."""
import os

import numpy as np
import pytest

import dense_scenarios as DS
from envelope_scenarios import census, check_census

pytestmark = pytest.mark.gpu

TOL_CERT = 1e-7     # N, whole horizon, against the oracle
TOL_FORMS = 2e-7    # N, whole horizon, dense against fused
TOL_H, TOL_G = 1e-13, 1e-12    # P0 (tests/test_gpu_parity.py)
SIZES = {10: (8192, (1, 2, 3, 4)), 20: (2048, (1, 2))}
SUBSET = 512
SEED = 211


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def engines(a1):
    e = {N: a1.Engine(a1.default_config(horizon=N)) for N in (10, 20)}
    yield e
    for x in e.values():
        x.close()


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _solve(torch, a1, eng, H, g, contact):
    """a1mpc_solve_dense_batch on device arrays; u and status start as NaN and -7, so a QP the solve never writes shows"""
    B, n = g.shape
    u = torch.full((B, n), float("nan"), dtype=torch.float64, device="cuda")
    status = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    a1._check(a1.lib().a1mpc_solve_dense_batch(eng.h, B, H.data_ptr(), g.data_ptr(), contact.data_ptr(), u.data_ptr(), status.data_ptr()))
    eng.sync()
    return u.cpu().numpy(), status.cpu().numpy()


def _chain(torch, a1, eng, d):
    """a1mpc_qp_mats_batch into a1mpc_solve_dense_batch, every array on the device: H, g, contact (device) and u, status (host)"""
    B = len(d["contact"])
    n = 12 * eng.cfg.horizon
    A_d, B_list, x0, x_d = (_dev(torch, d[k]) for k in ("A_d", "B_list", "x0", "x_d"))
    contact = _dev(torch, d["contact"].astype(np.int32))       # the masks are below 16: the same bits as uint32
    H = torch.empty((B, n, n), dtype=torch.float64, device="cuda")
    g = torch.empty((B, n), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    a1._check(a1.lib().a1mpc_qp_mats_batch(eng.h, B, A_d.data_ptr(), B_list.data_ptr(), x0.data_ptr(), x_d.data_ptr(), H.data_ptr(), g.data_ptr()))
    eng.sync()
    u, status = _solve(torch, a1, eng, H, g, contact)
    return H, g, contact, u, status


def _threads(O):
    return max(1, min(O.hardware_threads(), len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 1))


@pytest.mark.parametrize("name", DS.FAMILIES)
@pytest.mark.parametrize("horizon", [10, 20])
def test_per_step_chain_on_the_device(a1, O, torch, engines, horizon, name):
    B, counts = SIZES[horizon]
    ocfg = O.make_config(horizon=horizon)
    d = DS.build(a1, ocfg, name, B, SEED, counts)
    DS.check_bd_step(name, d)
    H, g, contact, u, status = _chain(torch, a1, engines[horizon], d)
    assert (status == a1.STATUS_OPTIMAL).all(), (np.bincount(status + 7), np.nonzero(status)[0][:10])
    idx = np.sort(np.random.default_rng([SEED, horizon, DS.FAMILIES.index(name)]).choice(B, SUBSET, replace=False))
    Ho, go = DS.qp_mats(O, ocfg, d, idx)
    ti = torch.from_numpy(idx).cuda()
    Hd, gd = H[ti].cpu().numpy(), g[ti].cpu().numpy()
    eH = (np.abs(Hd - Ho).max(axis=(1, 2)) / np.abs(Ho).max(axis=(1, 2))).max()
    eg = (np.abs(gd - go).max(axis=1) / np.abs(go).max(axis=1)).max()
    assert eH <= TOL_H and eg <= TOL_G, (eH, eg)
    uo, cert = DS.oracle_solve(O, ocfg, Ho, go, contact.cpu().numpy()[idx], nthreads=_threads(O))
    assert cert.all()
    check_census("%s N=%d" % (name, horizon), census(uo, d["contact"][idx]), DS.CENSUS_FLOORS[horizon])
    err = np.abs(u[idx] - uo).max(axis=1)
    ns = np.array([bin(int(c)).count("1") for c in d["contact"][idx]])
    print("%-9s N=%d B=%d: H %.1e g %.1e; worst |u - u*| per stance count: %s" % (
        name, horizon, B, eH, eg, "  ".join("%d: %.1e" % (k, err[ns == k].max()) for k in range(1, 5) if (ns == k).any())))
    assert err.max() <= TOL_CERT, (err.max(), int(idx[err.argmax()]))


@pytest.mark.parametrize("horizon,B", [(10, 2048), (20, 512)])
def test_dense_and_fused_forms_agree(a1, O, engines, horizon, B):
    """the same constant-B_d QP through the direct dense factor and through the fused solve (Kronecker form for one or two feet,
    wrench space for three and four): B QPs per family"""
    eng = engines[horizon]
    ocfg = O.make_config(horizon=horizon)
    worst = {}
    for name in DS.FAMILIES:
        st = DS.build(a1, ocfg, name, B, SEED + 1, SIZES[horizon][1])["st"]
        H, g, _, _ = eng.build_qp(st)
        u, status = eng.solve_dense(H, g, st["contact"])
        del H, g
        _, sf, _, uf = eng.solve(st, want_u=True)
        assert (status == a1.STATUS_OPTIMAL).all() and (sf == a1.STATUS_OPTIMAL).all(), (name, np.bincount(status), np.bincount(sf))
        err = np.abs(u - uf.T).max(axis=1)
        ns = np.array([bin(int(c)).count("1") for c in st["contact"]])
        worst[name] = {k: float(err[ns == k].max()) for k in range(1, 5) if (ns == k).any()}
        assert err.max() <= TOL_FORMS, (name, err.max(), int(err.argmax()))
    print("N=%d dense vs fused, worst per stance count: %s" % (horizon, worst))


@pytest.mark.parametrize("horizon", [10, 20])
def test_permuted_and_repeated_batches_are_bit_identical(a1, O, torch, engines, horizon):
    B, counts = SIZES[horizon]
    eng = engines[horizon]
    d = DS.build(a1, O.make_config(horizon=horizon), "combined", B, SEED + 2, counts)
    H, g, contact, u, status = _chain(torch, a1, eng, d)
    u2, s2 = _solve(torch, a1, eng, H, g, contact)
    assert np.array_equal(s2, status) and np.array_equal(u2, u)
    perm = np.random.default_rng(horizon).permutation(B)
    tp = torch.from_numpy(perm).cuda()
    up, sp = _solve(torch, a1, eng, H[tp].contiguous(), g[tp].contiguous(), contact[tp].contiguous())
    assert np.array_equal(sp, status[perm]) and np.array_equal(up, u[perm])


@pytest.mark.parametrize("horizon", [10, 20])
def test_input_contract(a1, O, torch, engines, horizon):
    """each case of dense_scenarios.CASES edits one QP of a clean batch, in every class's queue between good QPs"""
    B, counts = SIZES[horizon]
    eng = engines[horizon]
    d = DS.build(a1, O.make_config(horizon=horizon), "push", B, SEED + 3, counts)
    H, g, contact, u0, s0 = _chain(torch, a1, eng, d)
    assert (s0 == a1.STATUS_OPTIMAL).all()
    plan = DS.contract_plan(d["contact"])
    Hx, gx, cx = H.clone(), g.clone(), contact.clone()
    for b, case, _ in plan:
        Hb, gb = H[b].cpu().numpy(), g[b].cpu().numpy()
        c = DS.edit(case, Hb, gb, int(d["contact"][b]), horizon)
        Hx[b], gx[b], cx[b] = torch.from_numpy(Hb).cuda(), torch.from_numpy(gb).cuda(), int(c)
    del H, g
    u, status = _solve(torch, a1, eng, Hx, gx, cx)
    DS.check_contract(a1, u, status, u0, s0, plan)


def test_n20_three_and_four_feet_are_reported_unsupported(a1, O, torch, engines):
    eng = engines[20]
    ocfg = O.make_config(horizon=20)
    bad = DS.build(a1, ocfg, "tilt", 256, SEED + 4, (3, 4))
    ok = DS.build(a1, ocfg, "tilt", 256, SEED + 5, (1, 2))
    H, g, contact, u_ok, s_ok = _chain(torch, a1, eng, ok)
    Hb, gb, cb, _, _ = _chain(torch, a1, eng, bad)
    perm = np.random.default_rng(4).permutation(512)
    tp = torch.from_numpy(perm).cuda()
    u, status = _solve(torch, a1, eng, torch.cat([Hb, H])[tp].contiguous(), torch.cat([gb, g])[tp].contiguous(), torch.cat([cb, contact])[tp].contiguous())
    was_bad = perm < 256
    assert (status[was_bad] == a1.STATUS_NUMERICAL).all() and np.array_equal(u[was_bad], np.zeros_like(u[was_bad]))
    assert (s_ok == a1.STATUS_OPTIMAL).all()
    assert np.array_equal(status[~was_bad], s_ok[perm[~was_bad] - 256]) and np.array_equal(u[~was_bad], u_ok[perm[~was_bad] - 256])
