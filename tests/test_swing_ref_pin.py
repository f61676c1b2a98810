"""CPU: the oracle's restatement of generate_swing_legs_ctrl and compute_grf's terrain adaptation (oracle_swing_*) against the
reference's own code -- the committed vectors of tests/golden/swing_v1.npz on every tick, and, where oracle/_ref exists, the live
reference build on fresh scenarios (and the committed file against a re-run of that build)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import swing_oracle_py as SO  # noqa: E402
from oracle import ref_swing_py as R  # noqa: E402
from swing_scenarios import CPS, KD_RESET, KD_ROS, KP_RESET, KP_ROS, check_tick  # noqa: E402

DT = 0.0025


def load_swing_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "swing_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def replay_oracle(G, robots):
    """runs the oracle over the recorded inputs of `robots` (one weight set) and checks every tick; returns the worst errors"""
    ids = list(robots)
    B, T = len(ids), G["contacts"].shape[1]
    kp, kd = G["kp"][ids[0]], G["kd"][ids[0]]
    assert all(np.array_equal(G["kp"][r], kp) and np.array_equal(G["kd"][r], kd) for r in ids)
    sw = SO.Swing(B)
    worst = [0.0, 0.0]
    for t in range(T):
        g = lambda k: np.ascontiguousarray(G[k][ids, t].T)
        fk, con, cur, rc = sw.legs(CPS, DT, kp, kd, g("gait_counter"), G["plan_contacts"][ids, t], g("rot_z"), g("foot_pos_abs"),
                                   g("foot_pos_target_rel"), g("foot_force"))
        ref = np.zeros((9, B))
        pitch = sw.terrain(1, g("root_pos"), ref)
        ef, ea = check_tick((fk, con, rc, pitch, ref[1]), (g("f_kin"), G["contacts"][ids, t], g("foot_pos_recent_contact"), G["terrain_pitch"][ids, t],
                                                           G["root_euler_d1"][ids, t]), "tick %d" % t)
        assert np.abs(cur - g("foot_pos_cur")).max() <= 1e-15
        worst = [max(worst[0], ef), max(worst[1], ea)]
    return worst


def test_fixture_covers_what_it_must():
    G = load_swing_golden()
    assert G["contacts"].shape == (6, 300)
    assert (G["movement_mode"][:, 0] == 0).all() and (G["movement_mode"][:, -1] == 1).all()       # standstill, then trot
    assert len(np.unique(G["gait_counter_speed"][:, 0])) >= 3
    assert ((G["contacts"] & ~G["plan_contacts"]) != 0).any()                                      # early contacts
    e1 = G["root_euler_d1"]
    assert e1.max() == 0.5 and e1.min() == -0.5                                                    # both signs, clipped
    assert (G["root_pos"][:, :, 2] <= 0.1).any()
    assert np.array_equal(G["kp"][0], KP_RESET) and np.array_equal(G["kd"][0], KD_RESET)
    assert np.array_equal(G["kp"][5], KP_ROS) and np.array_equal(G["kd"][5], KD_ROS)


def test_oracle_matches_the_reference_vectors_on_every_tick():
    G = load_swing_golden()
    for robots in (range(0, 3), range(3, 6)):
        replay_oracle(G, robots)


def test_all_recent_contact_points_zero_give_angle_zero_exactly():
    """the exactly singular start (W^T W = diag(4, 0, 0)): the pseudo-inverse drops both zero singular values, the plane is flat"""
    sw = SO.Swing(4)
    pos = np.zeros((3, 4)); pos[2] = 0.3
    ref = np.full((9, 4), 7.0)
    for _ in range(3):
        pitch = sw.terrain(1, pos, ref)
        assert (pitch == 0.0).all() and (ref[1] == 0.0).all() and (ref[[0, 2, 3, 4, 5, 6, 7, 8]] == 7.0).all()


needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libref_swing.so absent (no /root/reference on this machine)")


@needs_ref
def test_golden_file_is_what_the_reference_build_produces():
    """re-run the committed inputs through the live reference build: every record bit-identical"""
    import make_swing_golden as M
    G = load_swing_golden()
    inp = {k: G[k] for k in M.INPUTS}
    inp["speed"] = G["gait_counter_speed"][:, 0]
    rec = M.run_reference(inp, G["kp"], G["kd"])
    for k, v in rec.items():
        assert np.array_equal(v, G[k]), k


@needs_ref
def test_oracle_equals_reference_build_on_fresh_scenarios():
    import make_swing_golden as M
    rng = np.random.default_rng(77)
    robots = [((rng.uniform(-1, 1), rng.uniform(-0.3, 0.3)), bool(rng.random() < 0.5), bool(rng.random() < 0.3), float(rng.choice([1.5, 2.0, 3.0, 4.0])))
              for _ in range(8)]
    inp = M.scenario(4242, robots, 300)
    for kp, kd, sel in ((KP_RESET, KD_RESET, range(0, 4)), (KP_ROS, KD_ROS, range(4, 8))):
        sub = {k: v[list(sel)] for k, v in inp.items()}
        rec = M.run_reference(sub, np.stack([kp] * 4), np.stack([kd] * 4))
        G = {k: sub[k] for k in M.INPUTS}
        G.update(rec, kp=np.stack([kp] * 4), kd=np.stack([kd] * 4))
        replay_oracle(G, range(4))
