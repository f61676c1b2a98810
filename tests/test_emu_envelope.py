"""The MPC solve on the states the controller produces outside the benchmark's trot distribution (tests/envelope_scenarios.py),
on the CPU emulator of the device code, every QP against the oracle's exact solver.

The wrench-space classes (three and four stance feet) used to end some of these QPs NUMERICAL although every input was finite and
the QP well posed: with a foot-step on an edge of the friction pyramid, the interior-point weights of its two active faces exceed
2R by ~1e16, and the cofactor inverse of its 3x3 block D = 2R + C'WC divided by a determinant that had cancelled to noise, zero or
a negative number.  The blocks are now inverted from an LDL' factor whose last pivot is formed from the multipliers
(WrenchLS::factor_fn, solve_qp); the QPs that failed are kept in tests/golden/envelope_numerical_n{10,20}.npz."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402
from envelope_scenarios import FAMILIES, census, check_census, family  # noqa: E402

TOL_CERT = 1e-7     # N: the engine's own figure for a certified QP

# a floor per census count, as a fraction of the QPs of a family (about half of what the families give at N = 10 and 20)
FLOORS = {
    "height": {"fzmax": 0.15, "vertex": 0.30, "edge": 0.30, "foot0": 0.15},
    "tilt": {"fzmax": 0.15, "vertex": 0.30, "edge": 0.50, "foot0": 0.08},
    "push": {"fzmax": 0.30, "vertex": 0.20, "edge": 0.50, "foot0": 0.12},
    "combined": {"fzmax": 0.30, "vertex": 0.25, "edge": 0.50, "foot0": 0.12},
}


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


def _check_family(E, a1, O, name, horizon, B, seed):
    st = family(a1, name, B, seed)
    fo, info, uo = O.compute_grf_batch(O.make_config(horizon=horizon), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
    check_census("%s N=%d" % (name, horizon), census(uo, st["contact"]), FLOORS[name])
    assert (info[:, 1] == 1).all()
    f, status, iters, _ = E.solve(a1.default_config(horizon=horizon), st)
    err = np.abs(f - fo).max(axis=0)
    assert (status == a1.STATUS_OPTIMAL).all(), (np.bincount(status), np.nonzero(status)[0][:10], st["contact"][status != 0][:10])
    assert err.max() <= TOL_CERT, (err.max(), int(err.argmax()))


@pytest.mark.parametrize("name", FAMILIES)
def test_envelope_family_n10(E, a1, O, name):
    _check_family(E, a1, O, name, 10, 384, 101)


@pytest.mark.parametrize("name", FAMILIES)
def test_envelope_family_n20(E, a1, O, name):
    _check_family(E, a1, O, name, 20, 128, 103)


@pytest.mark.parametrize("horizon", [10, 20])
def test_wrench_space_edge_pivots_are_not_numerical(E, a1, O, horizon):
    """The three- and four-stance QPs of the families (stream 101) that the wrench-space classes reported NUMERICAL: the interior
    point's factorisation of Hw^-1 + S failed because D^-1 of a foot-step on a friction edge came out Inf or 10 % off.  Every one
    is well posed (the oracle certifies it) and has a stance foot-step on a friction edge at the optimum; with the LDL' inverse
    each is certified and within 1e-7 N of the oracle."""
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "envelope_numerical_n%d.npz" % horizon)))
    assert all(bin(int(m)).count("1") >= 3 for m in d["contact"])          # the wrench-space classes
    fo, info, uo = O.compute_grf_batch(O.make_config(horizon=horizon), obatch(O, d), O.MODE_EXACT, nthreads=2, want_u=True)
    assert (info[:, 1] == 1).all()
    c = census(uo, d["contact"])
    assert c["edge"] == c["B"], c
    f, status, iters, _ = E.solve(a1.default_config(horizon=horizon), d)
    assert (status == a1.STATUS_OPTIMAL).all(), status
    assert np.abs(f - fo).max() < TOL_CERT, np.abs(f - fo).max()
