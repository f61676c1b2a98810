"""CPU tests of the a1mpc_stance_qp_batch kernels (stance_pack_kernel, stance_qp_kernel<NS>) on the block emulator (tests/emu/emu_stance.cpp),
in all three lane orders, against the restatement: the PD law of tests/stance_scenarios.py (root_acc within 1e-13 max(1, |acc|_inf): the
same dozen products and sums in another order) and the oracle's exact solve of the 12-variable QP (forces within 1e-4 N), with the
statuses exact.  The QP half must be the QP of a1mpc_grf_qp_batch: f_body and status bit-identical to the emulated grf_qp kernels fed the
same root_acc."""
import os

import numpy as np
import pytest

from stance_scenarios import NAMES, gains, oracle_forces, robots, root_acc_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORDERS = (0, 1, 2)   # lane order between collectives: ascending, descending, pseudo-random


@pytest.fixture(scope="module")
def E(built):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import emu_stance_py
    return emu_stance_py


@pytest.fixture(scope="module")
def EG(built):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import emu_py
    return emu_py


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def _golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "stance_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _check(E, EG, O, st, name, order):
    mass, kdl, kpa, kda = gains(name)
    args = [st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")]
    f, status, acc = E.stance_qp(*args, kdl, kpa, kda, mass, want_acc=True, order=order)
    acc0 = root_acc_batch(st["x0"], st["rot"], st["des"], st["kp_linear"], kdl, kpa, kda, mass)
    ea = float((np.abs(acc - acc0) / np.maximum(1.0, np.abs(acc0).max(axis=0))).max())
    assert ea <= 1e-13, ea
    f0, ok = oracle_forces(O, acc0, st["rot_z"], st["rot"], st["foot"], st["contact"])
    assert ok.all()
    expect = np.where(st["contact"] & 15 == 0, 4, 0)
    assert np.array_equal(status, expect), np.bincount(status)
    ef = float(np.abs(f - f0).max())
    assert ef <= 1e-4, ef
    # the same QP as a1mpc_grf_qp_batch, fed this call's own root_acc (QP-major)
    fg, sg = EG.grf_qp(acc.T, st["rot_z"].T, st["rot"].T, st["foot"].T, st["contact"], order=order)
    assert np.array_equal(fg.T, f) and np.array_equal(sg, status)
    return ea, ef


@pytest.mark.parametrize("order", ORDERS)
def test_emulator_matches_restatement_on_the_golden_states(E, EG, O, order):
    G = _golden()
    for y, name in enumerate(NAMES):
        sel = np.nonzero(G["yaml"] == y)[0]
        st = {k: np.ascontiguousarray(G[k][sel].T) for k in ("x0", "rot", "rot_z", "foot", "des", "kp_linear")}
        st["contact"] = G["contact"][sel]
        _check(E, EG, O, st, name, order)
        # and the reference's own forces (the stored ones carry the ADMM tolerance of the stand-in solver)
        f, status = E.stance_qp(*[st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")], *gains(name)[1:], gains(name)[0],
                                want_acc=False, order=order)
        assert np.abs(f.T - G["f_body"][sel]).max() <= 1e-4


@pytest.mark.parametrize("order", ORDERS)
def test_emulator_matches_restatement_on_random_robots(E, EG, O, order):
    B = 2048
    worst = [0.0, 0.0]
    for y, name in enumerate(NAMES):
        st = robots(B // 3 + 1, 400 + 10 * order + y, name)
        ea, ef = _check(E, EG, O, st, name, order)
        worst = [max(worst[0], ea), max(worst[1], ef)]
    print("order %d: root_acc rel %.1e, |f - f_oracle| %.1e N" % (order, *worst))


def test_emulator_bad_inputs(E, O):
    st = robots(64, 5, "hardware", contact=np.full(64, 15))
    st["contact"][7] = 0
    st["x0"][4, 11] = np.nan
    st["rot_z"][2, 20] = np.inf
    mass, kdl, kpa, kda = gains("hardware")
    f, status = E.stance_qp(*[st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")], kdl, kpa, kda, mass, want_acc=False)
    assert status[7] == 4 and status[11] == 3 and status[20] == 3
    assert (f[:, [7, 11, 20]] == 0.0).all()
    keep = np.setdiff1d(np.arange(64), [7, 11, 20])
    assert (status[keep] == 0).all()
