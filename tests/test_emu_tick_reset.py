"""CPU: the masked reset kernels of a control tick (tick_reset_robots_kernel, ekf_init_pending) on the block emulator.  Every state buffer is
filled with random values; after a masked reset the masked robots hold bit for bit what the whole-batch init kernels write (imu_init_kernel,
command_init_kernel with ref in MPC mode, swing_init_kernel) and zero x0, gait counters, tau and warm slot, and every word of the other
robots is unchanged.  The masked EKF init matches ekf_init_kernel on the flagged robots, leaves the rest alone and clears the flags."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_tick_reset_py as E  # noqa: E402

B = 300          # three blocks, the last one partial
N = 10           # the horizon whose tick keeps a warm slot


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def _bits(a):
    return a.view(np.uint8) if a.dtype == np.uint8 else a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _state(rng, S, variant, mpc, a1):
    r = lambda rows: rng.standard_normal((rows, B)) * 10.0
    st = dict(x0=r(12), gc=r(4), tau=r(12), imu=r(S["imu"]) if variant != a1.VARIANT_HARDWARE else None, cmd=r(S["cmd"]),
              ref=r(9) if mpc else None, swing=r(S["swing"]),
              warm=rng.integers(0, 2**32, B * (S["warm_hdr"] + 4 * N), dtype=np.uint32) if mpc else None)
    return {k: v for k, v in st.items() if v is not None}


def _masks(rng):
    some = lambda p: (rng.random(B) < p) * rng.integers(1, 256, B)   # any nonzero byte marks a robot
    return dict(none=np.zeros(B, np.uint8), all=np.ones(B, np.uint8), quarter=some(0.25).astype(np.uint8), one_pct=some(0.01).astype(np.uint8),
                bool_like=(rng.random(B) < 0.5).astype(np.uint8))


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("mode", ["qp", "mpc"])
def test_masked_reset_on_emulator(a1, variant, mode):
    mpc = mode == "mpc"
    tp = a1.default_tick_params(variant, a1.TICK_MPC if mpc else a1.TICK_QP)
    S = E.sizes()
    ww = S["warm_hdr"] + 4 * N
    rng = np.random.default_rng(100 + 10 * variant + mpc)
    # what the init kernels of a1mpc_tick_reset write, over random buffers
    init = _state(rng, S, variant, mpc, a1)
    E.init_kernels(B, tp.command, init.get("imu"), init["cmd"], init.get("ref"), init["swing"])
    for k in ("x0", "gc", "tau", "warm"):
        if k in init:
            init[k][...] = 0
    masks = _masks(rng)
    for name, mask in masks.items():
        for flag in (True, False):
            st = _state(rng, S, variant, mpc, a1)
            before = {k: v.copy() for k, v in st.items()}
            pending = rng.integers(0, 2, B).astype(np.uint8) if flag else None
            p0 = pending.copy() if flag else None
            E.reset_robots(B, mask, tp.command, st["x0"], st["gc"], st["tau"], st.get("imu"), st["cmd"], st.get("ref"), st["swing"], st.get("warm"),
                           ww, pending)
            m = mask != 0
            for k, v in st.items():
                if k == "warm":
                    v, w0, wi = v.reshape(B, ww).T, before[k].reshape(B, ww).T, init[k].reshape(B, ww).T
                else:
                    w0, wi = before[k], init[k]
                assert np.array_equal(_bits(v[:, m]), _bits(wi[:, m])), (name, k)
                assert np.array_equal(_bits(v[:, ~m]), _bits(w0[:, ~m])), (name, k)
            if flag:
                assert np.array_equal(pending, np.where(m, 1, p0).astype(np.uint8)), name   # several calls before a run: the union
    # the start values are not trivially zero, so the comparison above can tell a missed command field from a written one
    assert (init["cmd"] != 0).any() and masks["quarter"].any() and not masks["quarter"].all()


def test_masked_ekf_init_on_emulator(a1):
    S = E.sizes()
    rng = np.random.default_rng(7)
    ekf = rng.standard_normal((B, S["ekf"]))
    fpr, rot, x0 = rng.standard_normal((12, B)) * 0.3, rng.standard_normal((9, B)), rng.standard_normal((12, B))
    full = ekf.copy()
    E.ekf_init(B, full, fpr, rot)
    for p in (0.0, 0.3, 1.0):
        e, x = ekf.copy(), x0.copy()
        pending = ((rng.random(B) < p) * rng.integers(1, 256, B)).astype(np.uint8)
        m = pending != 0
        E.ekf_init_pending(B, pending, e, fpr, rot, x)
        assert np.array_equal(_bits(e[m]), _bits(full[m])) and np.array_equal(_bits(e[~m]), _bits(ekf[~m])), p
        est = [3, 4, 5, 9, 10, 11]
        other = [r for r in range(12) if r not in est]
        assert (x[est][:, m] == 0).all() and np.array_equal(_bits(x[est][:, ~m]), _bits(x0[est][:, ~m]))
        assert np.array_equal(_bits(x[other]), _bits(x0[other]))
        assert not pending.any()
