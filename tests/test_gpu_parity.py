"""Parity tests proper: the CUDA path (through the C ABI, via ctypes) against the CPU oracle and the committed
golden fixtures.  Tolerances (fp64, stated by BASELINE.json north_star / SURVEY 8c):
   P0 build  : |H - H_oracle|_max / |H|_max <= 1e-13 ; |g - g_oracle|_max / |g|_max <= 1e-12
   P1 solve  : |f_gpu - f*|_inf <= 1e-4 N  (f* = unique optimum, KKT-certified by the oracle)
"""
import ctypes as C

import numpy as np
import pytest

from common import check_feasible, golden_groups, load_golden, obatch
from gpu_helpers import discrete_model

pytestmark = pytest.mark.gpu

TOL_F = 1e-4      # N, north_star
TOL_H = 1e-13
TOL_G = 1e-12


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def engine_for(a1, hz, wk, **extra):
    return a1.Engine(a1.default_config(horizon=hz, mass=wk["mass"], inertia=list(wk["inertia"]), q=list(wk["q"]), r=list(wk["r"]), **extra))


def test_golden_fixtures(a1):
    """committed golden vectors: every stance pattern class, both weight sets, N = 10 and 20"""
    for hz, w, wk, st, f_gold in golden_groups():
        eng = engine_for(a1, hz, wk)
        f, status, iters = eng.solve(st)
        assert (status == a1.STATUS_OPTIMAL).all(), (hz, w, status)
        assert np.abs(f - f_gold).max() <= TOL_F, (hz, w, np.abs(f - f_gold).max())
        eng.close()


def test_reference_test_mpc_fixture(a1, O):
    """the reference's own standalone driver state (test/test_mpc.cpp:15-91)"""
    ocfg, ob = O.test_mpc_fixture()
    eng = a1.Engine(a1.default_config(mass=15.0, q=list(ocfg.q), r=list(ocfg.r)))
    f, status, iters, u = eng.solve(dict(x0=ob.x0, rot=ob.rot, foot=ob.foot, ref=ob.ref, contact=ob.contact), want_u=True)
    ka = load_golden()["test_mpc_fixture"]["survey_known_answer"]
    assert status[0] == 0
    assert np.abs(f[0:3, 0] - ka["FL"]).max() <= 1e-6 and np.abs(f[6:9, 0] - ka["RL"]).max() <= 1e-6
    assert np.abs(f[3:6, 0]).max() == 0 and np.abs(f[9:12, 0]).max() == 0
    fz = u[:, 0].reshape(10, 4, 3)[:, 0, 2]
    assert np.allclose(fz, [42.790, 45.687, 47.351, 47.826, 47.060, 44.906, 41.114, 35.317, 29.772, 18.588], atol=6e-4)
    eng.close()


def test_p0_build_parity(a1, O, gpu_engine):
    """ConvexMpc members (hessian, gradient, lb, ub) vs the literal dense restatement"""
    st = a1.gen_states(32, 2, 11)
    H, g, lb, ub = gpu_engine.build_qp(st)
    ocfg = O.make_config()
    ob = obatch(O, st)
    for b in range(32):
        Ho, go, Ao, lbo, ubo = O.build_qp(ocfg, ob, b)
        assert np.abs(H[b] - Ho).max() <= TOL_H * np.abs(Ho).max()
        assert np.abs(g[b] - go).max() <= TOL_G * np.abs(go).max()
        assert np.array_equal(lb[b], lbo) and np.array_equal(ub[b], ubo)


def test_p0_build_parity_n20(a1, O):
    eng = a1.Engine(a1.default_config(horizon=20))
    st = a1.gen_states(4, 2, 12)
    H, g, lb, ub = eng.build_qp(st)
    ocfg = O.make_config(horizon=20)
    for b in range(4):
        Ho, go, Ao, lbo, ubo = O.build_qp(ocfg, obatch(O, st), b)
        assert np.abs(H[b] - Ho).max() <= TOL_H * np.abs(Ho).max() and np.abs(g[b] - go).max() <= TOL_G * np.abs(go).max()
    eng.close()


@pytest.mark.parametrize("config_id,B", [(2, 1024), (4, 512)])
def test_p1_solve_parity_trot_batches(a1, O, gpu_engine, config_id, B):
    """BASELINE configs[1] (trot, N=10, batch 1024, fp64) and the wide-noise states of config 4: every QP against
    the KKT-certified optimum"""
    st = a1.gen_states(B, config_id, 21)
    f, status, iters, u = gpu_engine.solve(st, want_u=True)
    fo, info, uo = O.compute_grf_batch(O.make_config(), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
    assert (info[:, 1] == 1).all() and info[:, 2].max() <= 1e-12
    assert (status == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= TOL_F
    assert np.abs(u.T - uo).max() <= TOL_F            # the whole horizon, not only the first step
    check_feasible(u, 0.3, 180.0, st["contact"])


def test_p1_hardware_weights_and_single_foot_classes(a1, O):
    """well-conditioned weight set (config/hardware_a1_mpc.yaml) and the 1- and 3-stance-foot kernels"""
    wk = load_golden()["weights"]["hardware"]
    eng = engine_for(a1, 10, wk)
    st = a1.gen_states(256, 4, 31)
    pats = np.array([0b0001, 0b0010, 0b0100, 0b1000, 0b0111, 0b1011, 0b1101, 0b1110, 0b0011, 0b1100, 0b0101, 0b1010], dtype=np.uint32)
    st["contact"] = pats[np.arange(256) % len(pats)]
    f, status, iters = eng.solve(st)
    fo, info = O.compute_grf_batch(O.make_config(**wk), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (status == 0).all() and np.abs(f - fo).max() <= TOL_F
    eng.close()


def test_p1_horizon_20(a1, O):
    """long-horizon path (BASELINE config 3's horizon), fp64, every stance-count class"""
    eng = a1.Engine(a1.default_config(horizon=20))
    st = a1.gen_states(96, 2, 41)
    st["contact"][:8] = [0b0001, 0b0111, 0b1000, 0b1110, 0b0010, 0b1011, 0b0100, 0b1101]
    f, status, iters = eng.solve(st)
    fo, info = O.compute_grf_batch(O.make_config(horizon=20), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    # with the wrench-space reduction the 4-stance factor is 120 x 120 (not 240 x 240) and fits in shared memory
    assert (status == 0).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= TOL_F
    eng.close()


def test_edge_cases(a1, O, gpu_engine):
    st = a1.gen_states(64, 2, 51)
    st["contact"][0] = 0            # no stance foot: all forces pinned to zero (ConvexMpc.cpp:233,238)
    st["contact"][1] = 0b10000 | 0  # bits above the four legs are ignored
    st["x0"][5, 2] = np.nan         # NaN input -> status, zero force, neighbours unaffected
    st["foot"][3, 3] = np.inf
    f, status, iters = gpu_engine.solve(st)
    assert status[0] == a1.STATUS_NO_CONTACT and status[1] == a1.STATUS_NO_CONTACT and np.abs(f[:, :2]).max() == 0
    assert status[2] == a1.STATUS_NUMERICAL and status[3] == a1.STATUS_NUMERICAL and np.abs(f[:, 2:4]).max() == 0
    ok = np.arange(64) >= 4
    fo, info = O.compute_grf_batch(O.make_config(), obatch(O, st, slice(4, 64)), O.MODE_EXACT, nthreads=4)
    assert (status[ok] == 0).all() and np.abs(f[:, ok] - fo).max() <= TOL_F
    # B = 1
    one = {k: (v[:1] if k == "contact" else v[:, 5:6].copy()) for k, v in st.items()}
    one["contact"] = st["contact"][5:6].copy()
    f1, s1, _ = gpu_engine.solve(one)
    assert s1[0] == 0 and np.abs(f1[:, 0] - f[:, 5]).max() == 0
    # argument errors
    with pytest.raises(a1.A1MpcError):
        gpu_engine.solve_ptrs(0, a1.Inputs(), a1.Outputs())


def test_ragged_ld_and_device_pointers(a1, gpu_engine):
    """ld > B (a slice of a larger SoA allocation) through host pointers, and the asynchronous device-pointer path"""
    big = a1.gen_states(300, 2, 61)
    B, off = 200, 37
    f_ref, s_ref, _ = gpu_engine.solve({k: (v[off:off + B].copy() if k == "contact" else v[:, off:off + B].copy()) for k, v in big.items()})
    f = np.zeros((12, 300)); status = np.full(300, -7, dtype=np.int32)
    inp = a1.Inputs(big["x0"][:, off:].ctypes.data, big["rot"][:, off:].ctypes.data, big["foot"][:, off:].ctypes.data,
                    big["ref"][:, off:].ctypes.data, big["contact"][off:].ctypes.data, 300)
    out = a1.Outputs(f[:, off:].ctypes.data, status[off:].ctypes.data, None, None, 300)
    gpu_engine.solve_ptrs(B, inp, out)
    assert np.array_equal(f[:, off:off + B], f_ref) and np.array_equal(status[off:off + B], s_ref)
    assert (status[:off] == -7).all() and (status[off + B:] == -7).all() and np.abs(f[:, off + B:]).max() == 0
    d = a1.DeviceBatch(gpu_engine, B)
    d.upload({k: (v[off:off + B].copy() if k == "contact" else v[:, off:off + B].copy()) for k, v in big.items()})
    gpu_engine.solve_ptrs(B, d.inp, d.out)
    fd, sd = d.download()
    assert np.array_equal(fd, f_ref) and np.array_equal(sd, s_ref)
    d.free()


def test_full_size_properties(a1, gpu_engine):
    """size-independent properties at the full shard size of config 5 (32768 QPs per GPU):
    run-to-run determinism, permutation equivariance (a QP's result does not depend on its neighbours or its slot),
    feasibility of every force, exact zeros on swing feet, statuses all certified"""
    B = 32768
    st = a1.gen_states(B, 2, 71)
    f, status, iters, u = gpu_engine.solve(st, want_u=True)
    assert (status == 0).all()
    f2, status2, _ = gpu_engine.solve(st)
    assert np.array_equal(f, f2)
    perm = np.random.default_rng(0).permutation(B)
    stp = {k: (v[perm].copy() if k == "contact" else v[:, perm].copy()) for k, v in st.items()}
    fp, sp, _ = gpu_engine.solve(stp)
    assert np.array_equal(fp, f[:, perm])
    check_feasible(u, 0.3, 180.0, st["contact"])
    swing = np.array([[((int(c) >> leg) & 1) == 0 for c in st["contact"]] for leg in range(4)])
    assert np.abs(f.reshape(4, 3, B)[swing.nonzero()[0], :, swing.nonzero()[1]]).max() == 0
    # body z-force roughly carries the robot (12 kg): sanity of the physical scale
    Rz = st["rot"].reshape(3, 3, B)
    fw = np.einsum("ijb,ljb->lib", Rz, f.reshape(4, 3, B)).sum(axis=0)     # sum of world-frame forces
    assert 60 < np.median(fw[2]) < 300
    assert (iters % 100).max() <= 40


def test_qp_mats_general_rollout(a1, O, gpu_engine):
    """ConvexMpc::calculate_qp_mats with a different B_d per step (test/test_mpc.cpp:106-122)"""
    st = a1.gen_states(6, 2, 81)
    cfg = gpu_engine.cfg
    N = cfg.horizon
    Ads, Bls, x0s, xds = [], [], [], []
    rng = np.random.default_rng(3)
    for b in range(6):
        Ad, Bd, x0, xd = discrete_model(cfg, st, b)
        Bl = np.concatenate([Bd * (1.0 + 0.05 * i) + (1e-4 * rng.standard_normal(Bd.shape) if b % 2 else 0.0) for i in range(N)], axis=0)
        Ads.append(Ad); Bls.append(Bl); x0s.append(x0); xds.append(xd)
    H, g = gpu_engine.qp_mats(np.array(Ads), np.array(Bls), np.array(x0s), np.array(xds))
    ocfg = O.make_config()
    for b in range(6):
        Ho, go = O.qp_mats(ocfg, Ads[b], Bls[b], x0s[b], xds[b])
        assert np.abs(H[b] - Ho).max() <= TOL_H * np.abs(Ho).max() and np.abs(g[b] - go).max() <= TOL_G * np.abs(go).max()


def test_solve_dense_is_an_osqp_replacement(a1, O, gpu_engine):
    """OsqpEigen::Solver call sites: dense hessian + gradient + contact-gated bounds in, getSolution() out"""
    st = a1.gen_states(24, 4, 91)
    st["contact"][:6] = [0b0001, 0b0111, 0b1111, 0b0110, 0b1000, 0]
    H, g, lb, ub = gpu_engine.build_qp(st)
    u, status = gpu_engine.solve_dense(H, g, st["contact"])
    ocfg = O.make_config()
    for b in range(24):
        uo, info = O.solve_dense(ocfg, H[b], g[b], st["contact"][b], O.MODE_EXACT)
        if st["contact"][b] == 0:
            assert status[b] == a1.STATUS_NO_CONTACT and np.abs(u[b]).max() == 0
            continue
        assert status[b] == 0 and info[1] == 1
        assert np.abs(u[b] - uo).max() <= TOL_F


def test_grf_qp_branch(a1, O, gpu_engine):
    """config 1: compute_grf's QP branch (stance_leg_control_type == 0), 12 variables"""
    rng = np.random.default_rng(5)
    B = 64
    st = a1.gen_states(B, 2, 101)
    rot = st["rot"].T.copy()
    yaw = st["x0"][2]
    rot_z = np.stack([np.cos(yaw), -np.sin(yaw), 0 * yaw, np.sin(yaw), np.cos(yaw), 0 * yaw, 0 * yaw, 0 * yaw, 1 + 0 * yaw], axis=1)
    foot = st["foot"].T.copy()
    acc = np.stack([rng.normal(0, 20, B), rng.normal(0, 20, B), 12 * 9.8 + rng.normal(0, 30, B), rng.normal(0, 5, B), rng.normal(0, 5, B), rng.normal(0, 2, B)], axis=1)
    contact = st["contact"].copy()
    contact[:6] = [0b1111, 0b0001, 0b0111, 0, 0b1010, 0b1111]
    acc[5] = [400, -300, 2500, 50, -40, 10]          # saturates fz_max and the friction faces
    f, status = gpu_engine.grf_qp(acc, rot_z, rot, foot, contact)
    for b in range(B):
        fo, info = O.grf_qp_single(acc[b], rot_z[b], rot[b], foot[b], contact[b], O.MODE_EXACT)
        if contact[b] == 0:
            assert status[b] == a1.STATUS_NO_CONTACT and np.abs(f[b]).max() == 0
            continue
        assert status[b] == 0 and info[1] == 1, (b, status[b], info)
        assert np.abs(f[b] - fo).max() <= TOL_F, (b, np.abs(f[b] - fo).max())


def test_config4_contact_schedule_and_terrain_normals(a1, O, gpu_engine):
    """BASELINE config 4 -- an extension beyond the reference: per-step contact schedules (trot / bound / rotary gallop at a
    random phase), per-foot terrain normals, wide state noise.  Oracle = the restated literal problem generalised the same way
    (per-step bounds, pyramid rows acting on Rf^T f), KKT-certified."""
    B = 384
    st = a1.gen_states(B, 4, 131)
    sched, normals = a1.gen_schedule(B, 10, 4, 131)
    sched[:, 0] = 0                      # no contact anywhere in the horizon
    sched[:, 1] = 0b1111                 # all four feet all the time, tilted terrain only
    sched[1:, 2] = 0                     # contact in the first step only
    sched[0, 3] = 0                      # nobody in contact in the step whose force is returned
    f, status, iters, u = gpu_engine.solve_ext(st, sched, normals, want_u=True)
    fo, info, uo = O.compute_grf_batch_ext(O.make_config(), obatch(O, st), sched, normals, O.MODE_EXACT, nthreads=O.hardware_threads(), want_u=True)
    assert (info[:, 1] == 1).all() and info[:, 2].max() <= 1e-12
    assert status[0] == a1.STATUS_NO_CONTACT and np.abs(f[:, 0]).max() == 0
    assert (status[1:] == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= TOL_F and np.abs(u.T - uo).max() <= TOL_F
    assert np.abs(f[:, 3]).max() == 0
    # schedule only / normals only / neither (falls through to the plain path)
    f1, s1, _ = gpu_engine.solve_ext(st, sched, None)
    fo1, _ = O.compute_grf_batch_ext(O.make_config(), obatch(O, st), sched, None, O.MODE_EXACT, nthreads=O.hardware_threads())
    assert np.abs(f1 - fo1).max() <= TOL_F
    f2, s2, _ = gpu_engine.solve_ext(st, None, normals)
    fo2, _ = O.compute_grf_batch_ext(O.make_config(), obatch(O, st), None, normals, O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (s2 == 0).all() and np.abs(f2 - fo2).max() <= TOL_F
    f3, s3, _ = gpu_engine.solve_ext(st, None, None)
    f4, s4, _ = gpu_engine.solve(st)
    assert np.array_equal(f3, f4)
    # anisotropic r weights cannot be combined with tilted pyramids: loud error, not an approximation
    wk = load_golden()["weights"]["hardware"]
    eng = engine_for(a1, 10, wk)
    with pytest.raises(a1.A1MpcError, match="isotropic"):
        eng.solve_ext(st, None, normals)
    eng.close()


def test_joint_torques_next_row(a1, O, gpu_engine):
    """SURVEY 8f.1: A1RobotControl::compute_joint_torques (A1RobotControl.cpp:289-319), fed straight from the solver's forces"""
    B = 512
    st = a1.gen_states(B, 2, 121)
    f, status, _ = gpu_engine.solve(st)
    rng = np.random.default_rng(9)
    jac = (0.2 * np.eye(3).reshape(1, 3, 3, 1) + 0.15 * rng.standard_normal((4, 3, 3, B))).reshape(36, B)
    f_kin = 30.0 * rng.standard_normal((12, B))
    km = np.array([0.1, 0.1, 0.1]); tg = np.array([0.8, 0, 0, -0.8, 0, 0, 0.8, 0, 0, -0.8, 0, 0])
    prev = rng.standard_normal((12, B))
    f_kin[4, 7] = np.nan                      # a NaN result keeps the previous torque (A1RobotControl.cpp:314-317)
    st["contact"][7] = 0b1101
    tau = gpu_engine.joint_torques(f, f_kin, jac, st["contact"], km, tg, tau_prev=prev)
    for b in range(0, B, 7):
        to = O.joint_torques(f[:, b], f_kin[:, b], jac[:, b], st["contact"][b], km, tg, tau_prev=prev[:, b])
        assert np.allclose(tau[:, b], to, rtol=1e-10, atol=1e-10, equal_nan=True), b
    assert np.array_equal(tau[3:6, 7], prev[3:6, 7])      # swing leg 1 of robot 7: NaN force -> all three torques NaN -> kept


def test_update_plan_previous_row(a1, O, gpu_engine):
    """SURVEY 8f.2: A1RobotControl::update_plan (A1RobotControl.cpp:148-202) batched, plus the horizon contact schedule that the
    extended solve consumes; then the schedule is actually fed to a1mpc_solve_batch_ext"""
    B = 257
    rng = np.random.default_rng(11)
    st = a1.gen_states(B, 2, 141)
    gp = a1.default_gait_params(10)
    gc0 = rng.uniform(0, 240, (4, B)); gc0[:, 0] = [119.5, 239.0, 0.0, 120.0]
    gcs = rng.choice([1.4, 1.5, 2.0], (4, B))
    mode = (rng.uniform(size=B) < 0.8).astype(np.uint32)
    yaw = st["x0"][2]
    rot_z = np.stack([np.cos(yaw), -np.sin(yaw), 0 * yaw, np.sin(yaw), np.cos(yaw), 0 * yaw, 0 * yaw, 0 * yaw, 1 + 0 * yaw])
    lvd = st["ref"][5:8].copy(); lvd[0, :5] = [2.0, -2.0, 0.0, 0.3, -0.3]     # saturates the foothold limits
    gc, plan, sched, trel, tabs, tw = gpu_engine.update_plan(gp, gc0, gcs, mode, st["x0"][9:12], lvd, rot_z, st["rot"], st["x0"][3:6])
    for b in range(B):
        g1, p1, s1, r1, a1_, w1 = O.update_plan(gp, mode[b], gc0[:, b], gcs[:, b], st["x0"][9:12, b], lvd[:, b], rot_z[:, b], st["rot"][:, b], st["x0"][3:6, b])
        assert np.array_equal(gc[:, b], g1) and plan[b] == p1 and np.array_equal(sched[:, b], s1), b
        assert np.abs(trel[:, b] - r1).max() <= 1e-15 and np.abs(tabs[:, b] - a1_).max() <= 1e-15 and np.abs(tw[:, b] - w1).max() <= 1e-14
    assert (sched[0] == plan).all()
    f, status, _ = gpu_engine.solve_ext(st, sched, None)
    fo, info = O.compute_grf_batch_ext(O.make_config(), obatch(O, st), sched, None, O.MODE_EXACT, nthreads=O.hardware_threads())
    nocontact = (sched == 0).all(axis=0)          # random counters can put every foot in swing for the whole horizon
    assert (status[nocontact] == a1.STATUS_NO_CONTACT).all() and (status[~nocontact] == 0).all()
    assert np.abs(f - fo).max() <= TOL_F


def test_fp64_peak_probe_and_profile_api(a1, gpu_engine):
    assert 20.0 < gpu_engine.fp64_peak_tflops() < 80.0     # H100 SXM fp64 FMA pipe: 34 TFLOP/s on the data sheet
    st = a1.gen_states(512, 2, 111)
    gpu_engine.profile_begin(4)
    for _ in range(3):
        gpu_engine.solve(st)
    ms, n = gpu_engine.profile_end()
    assert n == 3 and ms[1] > 0 and ms[3] > 0 and ms[0] >= 0


def test_cpp_shims_mirror_of_test_mpc(built):
    """tests/cpp/test_mpc_b200.cpp: the reference's test_mpc.cpp call sequence on ConvexMpcBatch +
    A1RobotControlBatch::compute_grf (C++ host over the C ABI), checked against the known optimum"""
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "test_mpc_b200")
    assert os.path.exists(exe), "run make (host target)"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
