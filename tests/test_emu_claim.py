"""The work queue of the class kernels on the CPU block emulator: every CTA claims its first QPs when it starts (claim_qps).

With one host thread the emulator runs the blocks of a class one after the other, the way CTAs start when each waits for a free
SM: block 0 claims its slots' QPs, draws every other QP of the class as its slots finish, and every later block finds the counter
exhausted and leaves before its set-up.  The results must not depend on which block served a QP."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402


@pytest.fixture(scope="module")
def E():
    import emu_py
    emu_py.lib()
    return emu_py


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_py
    oracle_py.lib()
    return oracle_py


@pytest.mark.parametrize("horizon,B", [(10, 96), (20, 24)])   # 20: the direct classes run as teams of two warps
def test_blocks_started_in_sequence_one_block_drains_each_class(E, O, horizon, B):
    a1 = E.a1mpc
    st = a1.gen_states(B, 2, 29)
    pats = [1, 2, 4, 8, 3, 5, 6, 9, 10, 12, 7, 11, 13, 14, 15, 0]   # every class, several CTAs' worth of trot QPs
    st["contact"][:len(pats)] = pats
    cfg = a1.default_config(horizon=horizon)
    f, status, iters, u, _ = E.solve(cfg, st, order=0, nthreads=1, want_u=True)
    fo, info, uo = O.compute_grf_batch(O.make_config(horizon=horizon), obatch(O, st), mode=O.MODE_EXACT, nthreads=4, want_u=True)
    nc = st["contact"] == 0
    assert (status[nc] == a1.STATUS_NO_CONTACT).all() and (status[~nc] == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() < 1e-6 and np.abs(u - uo.T).max() <= 1e-4
    # the same batch with the blocks spread over host threads (they interleave and share each class): bit for bit
    g = E.solve(cfg, st, order=0, nthreads=8, want_u=True)
    assert np.array_equal(f, g[0]) and np.array_equal(status, g[1]) and np.array_equal(iters, g[2]) and np.array_equal(u, g[3])


def test_compact_schedule_kernel_blocks_started_in_sequence(E, O):
    a1 = E.a1mpc
    B = 48
    st = a1.gen_states(B, 4, 57)
    sched, normals = a1.gen_schedule(B, 10, 4, 57)
    cfg = a1.default_config(horizon=10)
    f, status, iters = E.solve_sched2(cfg, st, sched, normals, order=0, nthreads=1)
    fo, info = O.compute_grf_batch_ext(O.make_config(horizon=10), obatch(O, st), sched, normals, mode=O.MODE_EXACT, nthreads=4)
    assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() < 1e-7
    g = E.solve_sched2(cfg, st, sched, normals, order=0, nthreads=8)
    assert np.array_equal(f, g[0]) and np.array_equal(status, g[1]) and np.array_equal(iters, g[2])
