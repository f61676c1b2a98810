"""CPU tests of the QP-mode stance QP on terrain normals (a1mpc_stance_qp_batch_ext: stance_pack_kernel, stance_qp_ext_kernel<NS>) and of the
walking surface's normal without the terrain stage (a1mpc_surface_normals_batch: surface_normals_kernel), on the block emulator
(tests/emu/emu_stance_terrain.cpp):
  * with every normal exactly e_z, f_body, status and root_acc are bit-identical to stance_qp_kernel<NS> over all 16 contact masks of
    tests/stance_scenarios.robots, in the three configurations and three lane orders;
  * with tilted, unnormalised per-foot normals (tilts up to 0.6 rad, exactly 0.5 among them, random azimuths, lengths 0.5 to 2), every
    OPTIMAL robot is within 1e-4 N of the exact solve of oracle/stance_terrain_oracle.cpp and every stance force lies in its foot's
    terrain pyramid to 1e-9 N;
  * a NaN, Inf, zero or downward normal on a stance foot gives NUMERICAL and zero forces, the same on a swing foot changes nothing;
  * surface_normals_kernel writes terrain_normals_kernel's normals bit for bit over the 6 x 300 recorded ticks of tests/golden/swing_v1.npz
    and leaves the swing state bytewise as it was;
  * the oracle with e_z normals is oracle_grf_qp_single, bit for bit."""
import os
import sys

import numpy as np
import pytest

from stance_scenarios import NAMES, gains, robots, root_acc_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
ORDERS = (0, 1, 2)   # lane order between collectives: ascending, descending, pseudo-random
MU, FZ_MAX = 0.7, 180.0
TOL_ORACLE = 1e-4    # N, the tolerance of the world-z stance QP against the oracle
TOL_PYRAMID = 1e-9   # N
OPTIMAL, MAXITER, NUMERICAL, NO_CONTACT = 0, 2, 3, 4   # A1MPC_STATUS_*


@pytest.fixture(scope="module")
def E(built):
    import emu_stance_terrain_py
    return emu_stance_terrain_py


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


@pytest.fixture(scope="module")
def OT(built):
    from oracle import stance_terrain_oracle_py
    return stance_terrain_oracle_py


def _bits(a):
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _args(st):
    return [st[k] for k in ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")]


def ez_normals(B):
    n = np.zeros((12, B))
    n[2::3] = 1.0
    return n


def tilted_normals(B, seed, max_tilt=0.6):
    """[12,B] per-foot normals: tilts uniform in [0, max_tilt] with every 7th exactly 0.5 rad, random azimuths, lengths 0.5 to 2"""
    rng = np.random.default_rng(seed)
    tilt, az = rng.uniform(0.0, max_tilt, (4, B)), rng.uniform(-np.pi, np.pi, (4, B))
    tilt.reshape(-1)[::7] = 0.5
    length = rng.uniform(0.5, 2.0, (4, B))
    n = np.stack([np.sin(tilt) * np.cos(az), np.sin(tilt) * np.sin(az), np.cos(tilt)], axis=1) * length[:, None, :]   # [4,3,B]
    return np.ascontiguousarray(n.reshape(12, B))


def terrain_frames(normals):
    """T(n) of every foot, [B,4,3,3] (columns e0 e1 e2), from the normals [12,B] normalised: the rotation about z x n taking z to n"""
    B = normals.shape[1]
    n = normals.T.reshape(B, 4, 3)
    n = n / np.linalg.norm(n, axis=2, keepdims=True)
    nx, ny, nz = n[..., 0], n[..., 1], n[..., 2]
    k = 1.0 / (1.0 + nz)
    T = np.empty((B, 4, 3, 3))
    T[..., 0, 0], T[..., 0, 1], T[..., 0, 2] = 1 - nx * nx * k, -nx * ny * k, nx
    T[..., 1, 0], T[..., 1, 1], T[..., 1, 2] = -nx * ny * k, 1 - ny * ny * k, ny
    T[..., 2, 0], T[..., 2, 1], T[..., 2, 2] = -nx, -ny, nz
    return T


def pyramid_excess(f_body, rot, contact, normals):
    """largest violation (N) of |t_x|, |t_y| <= mu f_n and 0 <= f_n <= 180 over the stance feet, in T(n)^T f_world, per robot [B].  f_body =
    R^T f_world is solved for f_world rather than multiplied by R: the orientation stage of a tick does not normalise the quaternion, so
    its rot is orthogonal only to the rounding of the quaternion's norm"""
    B = f_body.shape[1]
    Rt = rot.T.reshape(B, 3, 3).transpose(0, 2, 1)
    fw = np.linalg.solve(Rt, f_body.T.reshape(B, 4, 3).transpose(0, 2, 1)).transpose(0, 2, 1)
    loc = np.einsum("blji,blj->bli", terrain_frames(normals), fw)               # T^T f_world
    t = np.maximum(np.abs(loc[..., 0]), np.abs(loc[..., 1])) - MU * loc[..., 2]
    ex = np.maximum(np.maximum(t, -loc[..., 2]), loc[..., 2] - FZ_MAX)
    stance = (contact[:, None] >> np.arange(4)[None, :]) & 1 == 1
    return np.where(stance, ex, -np.inf).max(axis=1)


def check_against_oracle(OT, f, status, acc, st, normals, what=""):
    """every stance robot OPTIMAL or MAXITER; every OPTIMAL one within TOL_ORACLE of the exact solve and inside its terrain pyramids ->
    (worst |f - f_oracle|, worst pyramid excess, MAXITER count)"""
    stance = (st["contact"] & 15) != 0
    assert (status[~stance] == NO_CONTACT).all() and (f[:, ~stance] == 0.0).all()
    assert np.isin(status[stance], [OPTIMAL, MAXITER]).all(), (what, np.bincount(status))
    f0, info = OT.grf_qp_batch_ext(acc, st["rot_z"], st["rot"], st["foot"], st["contact"], normals)
    assert (info[:, 1] == 1).all(), what
    opt = status == OPTIMAL
    ef = float(np.abs(f[:, opt] - f0[:, opt]).max()) if opt.any() else 0.0
    ep = float(pyramid_excess(f[:, opt], st["rot"][:, opt], st["contact"][opt], normals[:, opt]).max()) if opt.any() else 0.0
    assert ef <= TOL_ORACLE and ep <= TOL_PYRAMID, (what, ef, ep)
    return ef, ep, int((status == MAXITER).sum())


@pytest.mark.parametrize("order", ORDERS)
def test_ez_normals_are_the_world_z_stance_qp(E, order):
    B = 16 * 24
    for y, name in enumerate(NAMES):
        st = robots(B, 700 + 10 * order + y, name, contact=np.arange(B) % 16)
        mass, kdl, kpa, kda = gains(name)
        f0, s0, a0 = E.stance_qp(*_args(st), kdl, kpa, kda, mass, order=order)
        f1, s1, a1 = E.stance_qp(*_args(st), kdl, kpa, kda, mass, normals=ez_normals(B), order=order)
        assert np.array_equal(_bits(f1), _bits(f0)) and np.array_equal(s1, s0) and np.array_equal(_bits(a1), _bits(a0)), (name, order)
        assert (s0[st["contact"] & 15 != 0] == OPTIMAL).mean() > 0.99


@pytest.mark.parametrize("order", ORDERS)
def test_tilted_normals_against_the_oracle(E, OT, order):
    B = 600
    worst, nmax = [0.0, 0.0], 0
    for y, name in enumerate(NAMES):
        st = robots(B, 800 + 10 * order + y, name)
        nrm = tilted_normals(B, 900 + 10 * order + y)
        mass, kdl, kpa, kda = gains(name)
        f, status, acc = E.stance_qp(*_args(st), kdl, kpa, kda, mass, normals=nrm, order=order)
        acc0 = root_acc_batch(st["x0"], st["rot"], st["des"], st["kp_linear"], kdl, kpa, kda, mass)
        assert float((np.abs(acc - acc0) / np.maximum(1.0, np.abs(acc0).max(axis=0))).max()) <= 1e-13
        ef, ep, nm = check_against_oracle(OT, f, status, acc, st, nrm, name)
        worst, nmax = [max(worst[0], ef), max(worst[1], ep)], nmax + nm
        # the tilted pyramid changes the answer: the world-z solve of the same QPs differs
        fz, _, _ = E.stance_qp(*_args(st), kdl, kpa, kda, mass, order=order)
        assert np.abs(fz - f).max() > 1.0
    assert nmax <= 3 * B * 1e-3, nmax
    print("order %d: |f - f_oracle| %.1e N, pyramid excess %.1e N, MAXITER %d" % (order, worst[0], worst[1], nmax))


def test_invalid_normals(E):
    B = 64
    st = robots(B, 17, "gazebo", contact=np.full(B, 0b0111))
    mass, kdl, kpa, kda = gains("gazebo")
    nrm = tilted_normals(B, 18, 0.4)
    f0, s0, _ = E.stance_qp(*_args(st), kdl, kpa, kda, mass, normals=nrm)
    assert (s0 == OPTIMAL).all()
    poison = [(np.nan, 0.0, 1.0), (0.0, np.inf, 1.0), (0.0, 0.0, 0.0), (0.3, 0.0, -0.9), (1.0, 0.0, 0.0), (0.0, 0.0, -np.inf)]
    bad = nrm.copy()
    for i, v in enumerate(poison):
        leg = i % 3                                    # a stance foot
        bad[3 * leg:3 * leg + 3, 4 * i] = v
        bad[9:12, 4 * i + 1] = v                       # the swing foot (leg 3)
    f, s, _ = E.stance_qp(*_args(st), kdl, kpa, kda, mass, normals=bad)
    hit = np.arange(len(poison)) * 4
    assert (s[hit] == NUMERICAL).all() and (f[:, hit] == 0.0).all()
    rest = np.setdiff1d(np.arange(B), hit)
    assert np.array_equal(_bits(f[:, rest]), _bits(f0[:, rest])) and np.array_equal(s[rest], s0[rest])


def test_surface_normals_match_terrain_normals_on_the_golden_sequences(E):
    import emu_terrain_normals_py as TN
    from swing_scenarios import CPS
    from test_emu_terrain_normals import DT, load_swing_golden
    G = load_swing_golden()
    R, T = G["contacts"].shape
    groups = (range(0, 3), range(3, 6))
    state = TN.swing_init(R)
    sloped = 0
    for t in range(T):
        g = lambda k: np.ascontiguousarray(G[k][:, t].T)
        for grp in groups:
            sel = slice(grp[0], grp[-1] + 1)
            sub = np.ascontiguousarray(state[:, sel])
            TN.swing_legs(sub, CPS, DT, G["kp"][grp[0]], G["kd"][grp[0]],
                          *[np.ascontiguousarray(g(k)[..., sel]) for k in ("gait_counter", "plan_contacts", "rot_z", "foot_pos_abs",
                                                                           "foot_pos_target_rel", "foot_force")])
            state[:, sel] = sub
        pos = g("root_pos")
        before = state.copy()
        n1 = E.surface_normals(state, pos)
        assert np.array_equal(_bits(state), _bits(before)), t
        s0 = state.copy()
        _, n0, _ = TN.terrain_normals(s0, 1, pos, np.zeros((9, R)))
        assert np.array_equal(_bits(n1), _bits(n0)), t
        sloped += int((n1[2] < 1.0 - 1e-6).sum())
        state = s0                                     # the chain carries terrain_normals_kernel's filter on
    assert sloped > 0


def test_oracle_with_ez_normals_is_grf_qp_single(O, OT):
    B = 160
    st = robots(B, 31, "hardware", contact=np.arange(B) % 16)
    mass, kdl, kpa, kda = gains("hardware")
    acc = root_acc_batch(st["x0"], st["rot"], st["des"], st["kp_linear"], kdl, kpa, kda, mass)
    fb, info = OT.grf_qp_batch_ext(acc, st["rot_z"], st["rot"], st["foot"], st["contact"], ez_normals(B))
    for b in range(B):
        if st["contact"][b] & 15 == 0:
            continue
        f1, i1 = OT.grf_qp_single_ext(acc[:, b], st["rot_z"][:, b], st["rot"][:, b], st["foot"][:, b], int(st["contact"][b]), ez_normals(1)[:, 0])
        f0, i0 = O.grf_qp_single(acc[:, b], st["rot_z"][:, b], st["rot"][:, b], st["foot"][:, b], int(st["contact"][b]), O.MODE_EXACT)
        assert np.array_equal(_bits(f1), _bits(f0)) and np.array_equal(i1, i0) and np.array_equal(_bits(fb[:, b]), _bits(f0)), b
