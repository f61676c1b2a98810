"""OPTIMAL must mean optimal -- on the GPU, through the C ABI, EVERY QP of a batch against the oracle (not a sample), plus the QPs
that round 1's certificate got wrong (found on the CPU emulator after the round's GPU minutes were spent: stationarity on the
free coordinates was assumed after the linear solve).  Same checks as
tests/test_emu.py::test_certified_means_optimal_every_qp_checked."""
import os

import numpy as np
import pytest

from common import obatch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_F = 1e-4      # N, north_star gate; the engine's own figure is 1e-7


def test_gpu_certified_means_optimal_every_qp_checked(built):
    import a1mpc as a1
    from oracle import oracle_py as O
    eng = a1.Engine(a1.default_config(horizon=10))
    ocfg = O.make_config(horizon=10)
    nt = O.hardware_threads()
    d = dict(np.load(os.path.join(ROOT, "tools", "data", "false_certificates_r01.npz")))
    fo, info = O.compute_grf_batch(ocfg, obatch(O, d), O.MODE_EXACT, nthreads=2)
    f, status, iters = eng.solve(d)
    assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7, (status, np.abs(f - fo).max())
    for cid, seed in ((2, 31), (4, 32)):
        B = 32768
        st = a1.gen_states(B, cid, seed)
        st["contact"][:] = np.random.default_rng(seed).integers(1, 16, size=B).astype(np.uint32)
        fo, info = O.compute_grf_batch(ocfg, obatch(O, st), O.MODE_EXACT, nthreads=nt)
        f, status, iters = eng.solve(st)
        err = np.abs(f - fo).max(axis=0)
        assert (info[:, 1] == 1).all()
        assert (status == a1.STATUS_OPTIMAL).all(), np.bincount(status)
        assert err.max() <= TOL_F and (err > 1e-7).sum() == 0, (err.max(), int((err > 1e-7).sum()))
    eng.close()
