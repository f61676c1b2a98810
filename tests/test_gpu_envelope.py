"""-m gpu: the MPC solve through the C ABI on the states the controller produces outside the benchmark's trot distribution
(tests/envelope_scenarios.py: height commands over the whole clamp, terrain pitch references and tilted bodies, pushes, all of
them together; every stance mask), EVERY QP of every entry point against the oracle, with the checks of
tests/test_gpu_zy_certificate.py: every status OPTIMAL, max |f - f*| <= 1e-4 N and no QP more than 1e-7 N off.
tests/test_emu_envelope.py runs the same families on the CPU emulator, with the QPs that used to end NUMERICAL."""
import os

import numpy as np
import pytest

from common import load_golden, obatch
from envelope_scenarios import FAMILIES, census, check_census, family

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_F = 1e-4       # N, north_star gate
TOL_CERT = 1e-7    # N, the engine's own figure for a certified QP
ULP32_180 = float(np.spacing(np.float32(180.0)))
FLOORS = {"fzmax": 0.15, "vertex": 0.15, "edge": 0.30, "foot0": 0.08}   # fractions of the QPs; tests/test_emu_envelope.py has them per family


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def _engine(a1, horizon, wk=None, **extra):
    if wk is None:
        return a1.Engine(a1.default_config(horizon=horizon, **extra))
    return a1.Engine(a1.default_config(horizon=horizon, mass=wk["mass"], inertia=list(wk["inertia"]), q=list(wk["q"]), r=list(wk["r"]), **extra))


def _ocfg(O, horizon, wk=None):
    if wk is None:
        return O.make_config(horizon=horizon)
    return O.make_config(horizon=horizon, **wk)


def _check(a1, tag, f, status, fo, info):
    err = np.abs(f - fo).max(axis=0)
    assert (info[:, 1] == 1).all(), tag
    assert (status == a1.STATUS_OPTIMAL).all(), (tag, np.bincount(status))
    assert err.max() <= TOL_F and (err > TOL_CERT).sum() == 0, (tag, float(err.max()), int((err > TOL_CERT).sum()))


def _next_tick(st, rng):
    """one control tick later: the state moves by dt along its velocities, plus sensor-level noise (tests/test_gpu_warm.py)"""
    st2 = {k: v.copy() for k, v in st.items()}
    st2["x0"][3:6] += 0.0025 * st["x0"][9:12]
    st2["x0"][0:3] += 0.0025 * st["x0"][6:9]
    st2["x0"] += 0.03 * rng.standard_normal(st2["x0"].shape) * np.array([.02, .02, .02, .01, .01, .005, .1, .1, .1, .05, .05, .05])[:, None]
    return st2


@pytest.mark.parametrize("horizon,B", [(10, 4096), (20, 1024)])
def test_solve_batch_every_family(a1, O, horizon, B):
    eng = _engine(a1, horizon)
    for i, name in enumerate(FAMILIES):
        st = family(a1, name, B, 211 + i)
        f, status, iters = eng.solve(st)
        fo, info, uo = O.compute_grf_batch(_ocfg(O, horizon), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
        check_census("%s N=%d" % (name, horizon), census(uo, st["contact"]), FLOORS)
        _check(a1, (name, horizon), f, status, fo, info)
    eng.close()


def test_solve_batch_combined_hardware_weights(a1, O):
    wk = load_golden()["weights"]["hardware"]
    eng = _engine(a1, 10, wk)
    st = family(a1, "combined", 4096, 221)
    f, status, iters = eng.solve(st)
    fo, info = O.compute_grf_batch(_ocfg(O, 10, wk), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    _check(a1, "hardware", f, status, fo, info)
    eng.close()


def test_solve_batch_warm_over_ticks(a1, O):
    """a stored face can lead straight into the failing factorisation: every tick of every family against the oracle"""
    B, T = 2048, 4
    eng = _engine(a1, 10)
    ocfg = _ocfg(O, 10)
    rng = np.random.default_rng(9)
    for i, name in enumerate(FAMILIES):
        st = family(a1, name, B, 231 + i)
        warm = eng.warm_alloc(B)
        hits = []
        for t in range(T):
            f, status, iters = eng.solve_warm(st, warm)
            fo, info = O.compute_grf_batch(ocfg, obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
            _check(a1, (name, t), f, status, fo, info)
            hits.append(((iters % 100) == 0).mean())
            st = _next_tick(st, rng)
        assert hits[0] == 0.0 and min(hits[1:]) > 0.5, (name, hits)     # the later ticks do start from the stored faces
        a1.lib().a1mpc_device_free(eng.h, warm)
    eng.close()


def test_solve_batch_ext_and_ext_warm(a1, O):
    """a1mpc_gen_schedule schedules and terrain normals on the family states, cold and warm (schedules move one step per tick)"""
    B, N = 2048, 10
    eng = _engine(a1, N)
    ocfg = _ocfg(O, N)
    rng = np.random.default_rng(10)
    for i, name in enumerate(FAMILIES):
        st = family(a1, name, B, 241 + i)
        s_long, normals = a1.gen_schedule(B, N + 3, 4, 241 + i)
        sched = np.ascontiguousarray(s_long[:N])
        f, status, iters = eng.solve_ext(st, sched, normals)
        fo, info = O.compute_grf_batch_ext(ocfg, obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
        _check(a1, (name, "ext"), f, status, fo, info)
        warm = eng.warm_alloc(B)
        for t in range(3):
            sched = np.ascontiguousarray(s_long[t:t + N])
            f, status, iters = eng.solve_ext_warm(st, sched, normals, warm, shift=1)
            fo, info = O.compute_grf_batch_ext(ocfg, obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
            _check(a1, (name, "ext_warm", t), f, status, fo, info)
            st = _next_tick(st, rng)
        a1.lib().a1mpc_device_free(eng.h, warm)
    eng.close()


def test_precision32_combined(a1, O):
    """include/a1mpc.h, precision 32: the optimum of the QP posed by the fp32-rounded inputs, rounded to fp32"""
    B = 4096
    eng = _engine(a1, 10, precision=32)
    st = family(a1, "combined", B, 251)
    f, status, iters = eng.solve(st)
    eng.close()
    r = {k: (v if k == "contact" else v.astype(np.float32).astype(np.float64)) for k, v in st.items()}
    fo, info = O.compute_grf_batch(_ocfg(O, 10), obatch(O, r), O.MODE_EXACT, nthreads=O.hardware_threads())
    assert f.dtype == np.float32 and (status == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert (info[:, 1] == 1).all()
    err = float(np.abs(f.astype(np.float64) - fo).max())
    assert err <= 1e-4 + ULP32_180, err


def test_stance_qp_on_family_states(a1, O):
    """a1mpc_stance_qp_batch on the same states, the family's references as the desired state (gazebo QP gains), against the
    PD law and the oracle's QP (tests/stance_scenarios.py, as tests/test_gpu_stance.py::test_oracle_parity_65536 checks it)"""
    from stance_scenarios import YAMLS, gains, oracle_forces, root_acc_batch, rz_rows
    mass, kdl, kpa, kda = gains("gazebo")
    eng = a1.Engine(a1.default_config(mass=mass))
    B = 2048
    for i, name in enumerate(FAMILIES):
        st = family(a1, name, B, 261 + i)
        x0, ref = st["x0"], st["ref"]
        des = np.zeros((12, B))
        des[0:2] = ref[0:2]; des[2] = x0[2]; des[3:5] = x0[3:5]; des[5] = ref[8]
        des[6:9] = ref[5:8]; des[9:12] = ref[2:5]
        rot_z = rz_rows(x0[2])
        kpl = np.repeat(np.array(YAMLS["gazebo"][1])[:, None], B, axis=1)
        f, status, acc = eng.stance_qp(x0, st["rot"], rot_z, st["foot"], st["contact"], des, kpl, kdl, kpa, kda, want_acc=True)
        acc0 = root_acc_batch(x0, st["rot"], des, kpl, kdl, kpa, kda, mass)
        assert float((np.abs(acc - acc0) / np.maximum(1.0, np.abs(acc0).max(axis=0))).max()) <= 1e-13
        f0, ok = oracle_forces(O, acc0, rot_z, st["rot"], st["foot"], st["contact"])
        assert ok.all()
        opt = status == a1.STATUS_OPTIMAL
        # the stance QP's 40-iteration cap may leave a rare QP uncertified; it must say so, and never as NUMERICAL
        assert np.isin(status[~opt], [a1.STATUS_IPM_ONLY, a1.STATUS_MAXITER]).all() and (~opt).sum() <= B * 1e-3, (name, np.bincount(status))
        assert float(np.abs(f[:, opt] - f0[:, opt]).max()) <= TOL_F, name
    eng.close()


@pytest.mark.parametrize("horizon", [10, 20])
def test_wrench_space_edge_pivots_are_not_numerical(a1, O, horizon):
    """the QPs that the wrench-space classes reported NUMERICAL (a foot-step on a friction edge, its block of D inverted by
    cofactors; tests/test_emu_envelope.py has the story), on the GPU"""
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "envelope_numerical_n%d.npz" % horizon)))
    eng = _engine(a1, horizon)
    f, status, iters = eng.solve(d)
    eng.close()
    fo, info = O.compute_grf_batch(_ocfg(O, horizon), obatch(O, d), O.MODE_EXACT, nthreads=2)
    _check(a1, horizon, f, status, fo, info)
