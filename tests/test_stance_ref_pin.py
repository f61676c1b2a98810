"""The restatement of compute_grf's QP branch pinned to the REFERENCE'S OWN compiled code (CPU, no GPU): the PD law of
tests/stance_scenarios.py (and the one-robot tests/test_ref_pin.py::_root_acc) followed by the oracle's exact solve of the 12-variable QP.

tests/golden/stance_v1.npz was produced by oracle/_ref/libref_mpc.so (tests/golden/make_stance_golden.py).  On every stored state the
gradient -M^T Q root_acc matches the `q` the reference handed to OsqpEigen to 1e-13 relative (a dozen products summed in another order),
and the oracle's forces match the reference's within 2e-5 N: the stored forces are the OSQP-algorithm restatement's answer at eps 1e-11,
which along the flat directions of a few of these QPs stops up to 1.1e-5 N short of the optimum (measured; the same effect as the 2e-5 N
of tests/test_ref_pin.py::test_oracle_grf_qp_matches_reference_golden).
Where the reference sources were present at build time the same is run live on fresh states; there the forces are held to 1e-4 N, like
the live MPC check of test_ref_pin.py (measured 2.5e-5 N on the fresh states, the same ADMM tolerance)."""
import numpy as np
import pytest

from oracle import ref_py as R
from stance_scenarios import NAMES, YAMLS, gains, oracle_forces, qp_gradient, robots, root_acc_batch, to_ref9
from test_ref_pin import _root_acc

ROOT_TESTS = __import__("os").path.dirname(__import__("os").path.abspath(__file__))


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def _golden():
    import os
    with np.load(os.path.join(ROOT_TESTS, "golden", "stance_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _relerr(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_golden_covers_what_it_claims():
    G = _golden()
    assert len(G["yaml"]) == 96 and sorted(set(G["yaml"].tolist())) == [0, 1, 2]
    for y in range(3):
        sel = G["yaml"] == y
        assert sorted(set(G["contact"][sel].tolist())) == list(range(16))
        assert G["mass"][sel][0] == YAMLS[NAMES[y]][0]
    err = G["des"][:, 2] - G["x0"][:, 2]
    thr = 1.5 * 3.1415926
    assert (err > thr).any() and (err < -thr).any() and np.min(np.abs(np.abs(err) - thr)) > 1e-9
    assert (G["kp_linear"][:, :2] == 0).all(axis=1).sum() >= 32
    assert np.abs(G["x0"][:, :2]).max() <= 0.3


def test_restatement_matches_reference_golden(O):
    G = _golden()
    worst = dict(q=0.0, f=0.0, acc=0.0)
    for y, name in enumerate(NAMES):
        sel = np.nonzero(G["yaml"] == y)[0]
        mass, kdl, kpa, kda = gains(name)
        st = {k: np.ascontiguousarray(G[k][sel].T) for k in ("x0", "rot", "rot_z", "foot", "des", "kp_linear")}
        acc = root_acc_batch(st["x0"], st["rot"], st["des"], st["kp_linear"], kdl, kpa, kda, mass)
        for k, i in enumerate(sel):
            # the vectorised PD law is the one-robot statement of test_ref_pin.py
            g12 = np.concatenate([G["kp_linear"][i], kdl, kpa, kda])
            a1 = _root_acc(G["x0"][i].copy(), G["rot"][i], G["des"][i], g12, mass)
            worst["acc"] = max(worst["acc"], float(np.abs(a1 - acc[:, k]).max() / max(1.0, np.abs(a1).max())))
            worst["q"] = max(worst["q"], _relerr(qp_gradient(G["rot_z"][i], G["foot"][i], acc[:, k]), G["q"][i]))
        f, ok = oracle_forces(O, acc, st["rot_z"], st["rot"], st["foot"], G["contact"][sel])
        assert ok.all()
        worst["f"] = max(worst["f"], float(np.abs(f.T - G["f_body"][sel]).max()))
    assert worst["acc"] <= 1e-15 and worst["q"] <= 1e-13 and worst["f"] <= 2e-5, worst


needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libref_mpc.so absent (built only where the reference sources are)")


@needs_ref
def test_restatement_matches_reference_build_on_fresh_states(O):
    worst = dict(q=0.0, f=0.0)
    for y, name in enumerate(NAMES):
        B = 24
        st = robots(B, 900 + y, name)
        mass, kdl, kpa, kda = gains(name)
        acc = root_acc_batch(st["x0"], st["rot"], st["des"], st["kp_linear"], kdl, kpa, kda, mass)
        f, ok = oracle_forces(O, acc, st["rot_z"], st["rot"], st["foot"], st["contact"])
        assert ok.all()
        cfg = O.make_config(mass=mass)
        for b in range(B):
            ref9, yaw_d, pdxy = to_ref9(st["des"][:, b])
            r = R.compute_grf(cfg, st["x0"][:, b], st["rot"][:, b], st["foot"][:, b], ref9, int(st["contact"][b]), control_type=0, solver="tight",
                              rot_z=st["rot_z"][:, b], root_pos_d_xy=pdxy, yaw_d=yaw_d, gains=np.concatenate([st["kp_linear"][:, b], kdl, kpa, kda]))
            worst["q"] = max(worst["q"], _relerr(qp_gradient(st["rot_z"][:, b], st["foot"][:, b], acc[:, b]), r["qp"][1]))
            worst["f"] = max(worst["f"], float(np.abs(f[:, b] - r["f_body"]).max()))
    assert worst["q"] <= 1e-13 and worst["f"] <= 1e-4, worst


@needs_ref
def test_golden_file_is_what_the_reference_build_produces():
    G = _golden()
    from oracle import oracle_py as O_
    for i in (0, 17, 40, 95):
        name = NAMES[int(G["yaml"][i])]
        _, kdl, kpa, kda = gains(name)
        ref9, yaw_d, pdxy = to_ref9(G["des"][i])
        r = R.compute_grf(O_.make_config(mass=float(G["mass"][i])), G["x0"][i], G["rot"][i], G["foot"][i], ref9, int(G["contact"][i]), control_type=0,
                          solver="tight", rot_z=G["rot_z"][i], root_pos_d_xy=pdxy, yaw_d=yaw_d, gains=np.concatenate([G["kp_linear"][i], kdl, kpa, kda]))
        assert np.array_equal(r["qp"][1], G["q"][i]) and np.array_equal(r["f_body"], G["f_body"][i])
