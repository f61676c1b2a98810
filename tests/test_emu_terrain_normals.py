"""CPU: terrain_normals_kernel (a1mpc_terrain_normals_batch, and stage 7 of a tick whose pyramids stand on the estimated terrain) on the
block emulator, over the recorded sequences of tests/golden/swing_v1.npz (standstill then trot, slopes of both signs up to the 0.5 rad
clip, body heights <= 0.1 m).  Every tick, from the same swing state:
  * ref row 1, terrain_pitch and every word of the swing state are bit-identical to terrain_pitch_kernel's;
  * the normals are within 1e-13 of a numpy restatement of their definition from the recent-contact points (plane normal
    (-a1, -a2, 1) / |.|, tilt clipped to 0.5 rad, e_z while the body is low), away from the pseudo-inverse cutoff;
  * all four feet get the same normal, n_z >= cos 0.5, and with contacts the held schedule holds them in all N rows.
Also the clip, the low body and the all-zero start (n = e_z) on their own."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_terrain_normals_py as E  # noqa: E402
from swing_scenarios import CPS  # noqa: E402

DT = 0.0025
TOL_N = 1e-13
EPS = np.finfo(np.float64).eps


def load_swing_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "swing_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def _bits(a):
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def restated_normals(rc, root_z):
    """numpy restatement of the normal from foot_pos_recent_contact rc [12,B] and root_pos z [B] -> (normals [3,B], margin [B]); margin
    is the distance of W^T W's eigenvalues from the reference's pseudo-inverse cutoff eps * 3 * max|l|, as a ratio (inf when a
    singular value is exactly zero, which both sides drop)"""
    B = rc.shape[1]
    n = np.zeros((3, B))
    margin = np.full(B, np.inf)
    for b in range(B):
        x, y, z = rc[0::3, b], rc[1::3, b], rc[2::3, b]
        W = np.stack([np.ones(4), x, y], axis=1)
        lam, V = np.linalg.eigh(W.T @ W)
        v = W.T @ z
        tol = EPS * 3.0 * np.abs(lam).max()
        a = np.zeros(3)
        for k in range(3):
            if abs(lam[k]) > tol:
                a += V[:, k] * (V[:, k] @ v) / lam[k]
            if lam[k] != 0.0:
                margin[b] = min(margin[b], max(abs(lam[k]) / tol, tol / abs(lam[k])))
        m = np.array([-a[1], -a[2], 1.0])
        nb = m / np.linalg.norm(m)
        if np.arccos(nb[2]) > 0.5:
            nb = np.array([np.sin(0.5) * nb[0] / np.hypot(nb[0], nb[1]), np.sin(0.5) * nb[1] / np.hypot(nb[0], nb[1]), np.cos(0.5)])
        if not root_z[b] > 0.1:
            nb = np.array([0.0, 0.0, 1.0])
        n[:, b] = nb
    return n, margin


def _check_layout(normals, N=None, sched=None, contacts=None):
    assert np.array_equal(normals, np.tile(normals[0:3], (4, 1)))
    assert (normals[2] >= np.cos(0.5) - 1e-15).all()
    assert np.abs(np.linalg.norm(normals[0:3], axis=0) - 1.0).max() <= 4 * EPS
    if sched is not None:
        assert sched.shape == (N, contacts.shape[0]) and (sched == contacts[None, :]).all()


def test_golden_sequences_match_terrain_pitch_and_the_restatement():
    adapt = 1
    G = load_swing_golden()
    R, T = G["contacts"].shape
    N = 10
    groups = (range(0, 3), range(3, 6))            # the two gain sets of the fixture; the terrain stage does not read them
    assert all(np.array_equal(G["kp"][r], G["kp"][grp[0]]) and np.array_equal(G["kd"][r], G["kd"][grp[0]]) for grp in groups for r in grp)
    state = E.swing_init(R)
    worst, compared, seen = 0.0, 0, dict(clip=0, low=0, sloped=0)
    for t in range(T):
        g = lambda k: np.ascontiguousarray(G[k][:, t].T)
        con = np.zeros(R, dtype=np.uint32)
        for grp in groups:
            sel = slice(grp[0], grp[-1] + 1)
            sub = np.ascontiguousarray(state[:, sel])
            con[sel], _ = E.swing_legs(sub, CPS, DT, G["kp"][grp[0]], G["kd"][grp[0]],
                                       *[np.ascontiguousarray(g(k)[..., sel]) for k in ("gait_counter", "plan_contacts", "rot_z", "foot_pos_abs",
                                                                                        "foot_pos_target_rel", "foot_force")])
            state[:, sel] = sub
        assert np.array_equal(con, G["contacts"][:, t]), t
        rc = state[36:48].copy()
        assert np.array_equal(rc, g("foot_pos_recent_contact")), t
        pos = g("root_pos")
        s0, s1 = state.copy(), state.copy()
        ref0, ref1 = np.full((9, R), 3.0), np.full((9, R), 3.0)
        p0 = E.terrain_pitch(s0, adapt, pos, ref0)
        p1, nrm, sched = E.terrain_normals(s1, adapt, pos, ref1, contacts=con, N=N)
        assert np.array_equal(_bits(s1), _bits(s0)) and np.array_equal(_bits(ref1), _bits(ref0)) and np.array_equal(_bits(p1), _bits(p0)), t
        if adapt:
            assert np.abs(ref1[1] - G["root_euler_d1"][:, t]).max() <= 1e-7
        _check_layout(nrm, N, sched, con)
        want, margin = restated_normals(rc, pos[2])
        ok = margin > 1e6
        if ok.any():
            worst = max(worst, float(np.abs(nrm[0:3, ok] - want[:, ok]).max()))
            compared += int(ok.sum())
        seen["clip"] += int((ok & (pos[2] > 0.1) & (np.abs(nrm[2] - np.cos(0.5)) < 1e-15)).sum())
        seen["low"] += int((pos[2] <= 0.1).sum())
        seen["sloped"] += int((ok & (pos[2] > 0.1) & (nrm[2] < 1.0 - 1e-6) & (nrm[2] > np.cos(0.5) + 1e-6)).sum())
        state = s0
    print("%d of %d robot-ticks compared, worst |n - n_numpy| %.2e; %s" % (compared, R * T, worst, seen))
    assert worst <= TOL_N
    assert compared >= 0.9 * R * T
    assert seen["clip"] > 0 and seen["low"] > 0 and seen["sloped"] > 0, seen


def _state_with_points(points):
    """a swing state whose recent-contact points are points [B,4,3] (the rest of the state zero)"""
    B = points.shape[0]
    state = E.swing_init(B)
    state[36:48] = points.reshape(B, 12).T
    return state


def test_clip_low_body_and_zero_start():
    rng = np.random.default_rng(5)
    B = 64
    base = np.array([[0.17, 0.15], [0.17, -0.15], [-0.17, 0.15], [-0.17, -0.15]])
    # planes z = a0 + a1 x + a2 y with tilts from 0 to 1.2 rad in every direction
    tilt, az = rng.uniform(0.0, 1.2, B), rng.uniform(-np.pi, np.pi, B)
    a1, a2 = np.tan(tilt) * np.cos(az), np.tan(tilt) * np.sin(az)
    a0 = rng.uniform(-0.4, -0.2, B)
    pts = np.zeros((B, 4, 3))
    pts[:, :, 0:2] = base[None] + 0.01 * rng.standard_normal((B, 4, 2))
    pts[:, :, 2] = a0[:, None] + a1[:, None] * pts[:, :, 0] + a2[:, None] * pts[:, :, 1]
    pos = np.zeros((3, B))
    pos[2] = np.where(np.arange(B) % 4 == 3, 0.08, 0.3)
    pos[2, 7] = 0.1                                            # exactly at the threshold: low
    state = _state_with_points(pts)
    ref = np.zeros((9, B))
    _, nrm, _ = E.terrain_normals(state, 1, pos, ref)
    _check_layout(nrm)
    # without terrain adaptation: ref untouched, the rest as terrain_pitch_kernel, the same normals
    s0, s1, ref0, ref1 = _state_with_points(pts), _state_with_points(pts), np.full((9, B), 3.0), np.full((9, B), 3.0)
    p0 = E.terrain_pitch(s0, 0, pos, ref0)
    p1, n1, _ = E.terrain_normals(s1, 0, pos, ref1)
    assert (ref1 == 3.0).all() and (ref0 == 3.0).all() and np.array_equal(_bits(p1), _bits(p0)) and np.array_equal(_bits(s1), _bits(s0))
    assert np.array_equal(n1, nrm)
    low = pos[2] <= 0.1
    assert (nrm[0:3, low] == np.array([[0.0], [0.0], [1.0]])).all()
    hi = ~low
    m = np.stack([-a1, -a2, np.ones(B)])
    want = m / np.linalg.norm(m, axis=0)
    clip = hi & (tilt > 0.5)
    want[:, clip] = np.stack([np.sin(0.5) * np.cos(az[clip] + np.pi), np.sin(0.5) * np.sin(az[clip] + np.pi), np.full(clip.sum(), np.cos(0.5))])
    assert np.abs(nrm[0:3, hi] - want[:, hi]).max() <= 1e-12
    assert clip.sum() >= 8 and (hi & ~clip).sum() >= 8 and low.sum() >= 8
    # the clipped normal keeps the downhill direction: (n_x, n_y) points against the gradient (a1, a2)
    assert (nrm[0, clip] * a1[clip] + nrm[1, clip] * a2[clip] < 0).all()
    # the all-zero start: W^T W = diag(4, 0, 0), both zero singular values dropped, the plane is flat
    state = E.swing_init(B)
    ref = np.zeros((9, B))
    pitch, nrm, _ = E.terrain_normals(state, 1, np.tile([[0.0], [0.0], [0.3]], (1, B)), ref)
    assert (nrm[0:3] == np.array([[0.0], [0.0], [1.0]])).all() and (pitch == 0.0).all() and (ref[1] == 0.0).all()
