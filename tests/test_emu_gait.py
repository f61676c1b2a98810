"""CPU: the per-robot gait kernels (a1mpc_gait.cuh) on the block emulator.
  * With trot rows (240 / 120, offsets 0 120 120 0) the gait twins of the tick's front stage (tick_front_b_gait, tick_front_sched_gait) and
    the staged gait kernels (update_plan_gait_kernel, swing_legs_gait_kernel) are bit-identical to the plain tick_front_b / tick_front_sched
    in every array they write (counters, swing state, f_kin, contacts, schedule, kinematics), over 30 ticks of standstill -> walking ->
    toggled out and back, for the three adapter variants, held and scheduled, with integer and non-integer gait speeds.  The same holds for
    the uniform pair 200 / 100 (offsets 0 120 120 0) against the plain kernels given that pair.
  * update_plan_gait_kernel and swing_legs_gait_kernel with trot rows reproduce update_plan_kernel and swing_legs_kernel over the recorded
    ticks of tests/golden/swing_v1.npz, bit for bit, and a mixed batch of the five gaits matches a numpy restatement of the generalised
    counters, plan and schedule exactly.
  * Contact patterns over a full cycle at equal leg speeds: trot, pace and bound keep their pairs in phase, pronk has all feet down or
    none, the walk keeps three or four feet down, swings each leg once per cycle, in the order RL, FL, RR, FR.
  * The row check's rules and a1mpc_gait_row's table."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_command_py as EC  # noqa: E402
import emu_gait_py as EG  # noqa: E402
import emu_tick_py as E  # noqa: E402
from command_scenarios import DT  # noqa: E402
from tick_scenarios import tick_inputs  # noqa: E402

TABLE = {1: [0, 120, 120, 0, 240, 120], 2: [0, 120, 0, 120, 240, 120], 3: [0, 0, 120, 120, 240, 120], 4: [0, 0, 0, 0, 240, 120],
         5: [120, 0, 180, 60, 240, 180]}


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def rows_of(types):
    return np.ascontiguousarray(np.array([TABLE[int(t)] for t in types], dtype=np.float64).T)


def _sides(a1, tp, B, N, n):
    cp = tp.command
    imu = tp.command.variant != a1.VARIANT_HARDWARE
    sides = []
    for _ in range(n):
        z = lambda r: np.zeros((r, B))
        s = dict(rot=z(9), rz=z(9), x0=z(12), ia=z(3), ig=z(3), kpl=z(3), ref=z(9), des=z(12), fpr=z(12), jac=z(36), fvr=z(12), foot=z(12),
                 fk=z(12), gc=z(4), mode=np.zeros(B, dtype=np.uint32), contacts=np.zeros(B, dtype=np.uint32),
                 sched=np.zeros((N, B), dtype=np.uint32) if N else None, swing=z(EG.swing_fields()))
        s["imu"] = EC.imu_init(B) if imu else None
        s["cmd"] = EC.command_init(B, cp.variant, cp.body_height, cp.body_height_min, cp.body_height_max, np.array(cp.kp_linear),
                                   np.array(cp.kp_linear_lock), ref=s["ref"])
        sides.append(s)
    return sides


def run_fronts(a1, tp, gait, B, T, N, seed, speed=None, kinds=(EG.PLAIN, EG.TWIN, EG.STAGED)):
    """the tick's first stages on the emulator, one side per kind of front stage; every array of every side compared after every tick"""
    seqs, sp = tick_inputs(B, T, seed)
    speed = sp if speed is None else speed
    rng = np.random.default_rng(seed + 1)
    sides = _sides(a1, tp, B, N, len(kinds))
    plan, trel = np.zeros(B, dtype=np.uint32), np.zeros((12, B))
    for t in range(T):
        est = np.concatenate([np.array([0.0, 0.0, 0.28])[:, None] + 0.02 * rng.standard_normal((3, B)), 0.3 * rng.standard_normal((3, B))])
        pitch = rng.uniform(-0.3, 0.3, B)
        for kind, s in zip(kinds, sides):
            s["x0"][3:6], s["x0"][9:12] = est[:3], est[3:]
            s["ref"][1] = pitch
            E.front_a(False, B, DT, seqs["quat"][t], seqs["gyro"][t], seqs["acc"][t], s["imu"], s["rot"], s["rz"], s["x0"], s["ia"], s["ig"],
                      s["cmd"], seqs["cmd"][t], s["mode"], s["kpl"], s["ref"], s["des"])
            lvd = np.ascontiguousarray(s["ref"][5:8])
            EG.front(kind, B, tp, DT, N, gait, seqs["joint_pos"][t], seqs["joint_vel"][t], s["rot"], s["rz"], s["x0"], lvd, s["mode"], s["gc"], speed,
                     s["swing"], seqs["foot_force"][t], s["fpr"], s["jac"], s["fvr"], s["foot"], s["fk"], s["contacts"], s["sched"], plan, trel)
        for s in sides[1:]:
            for k in s:
                if s[k] is not None:
                    assert s[k].tobytes() == sides[0][k].tobytes(), (t, k)
    return sides[0]


@pytest.mark.parametrize("speeds", ["integer", "fractional"])
@pytest.mark.parametrize("N", [0, 10])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_trot_rows_reproduce_the_plain_front(a1, variant, N, speeds):
    B, T = 128, 26
    tp = a1.default_tick_params(variant, a1.TICK_MPC)
    tp.gait.horizon = N
    speed = None
    if speeds == "fractional":
        speed = np.ascontiguousarray(np.repeat(np.random.default_rng(5 + variant).uniform(1.5, 4.5, B)[None, :], 4, axis=0))
    s = run_fronts(a1, tp, rows_of([1] * B), B, T, N, 23 + variant, speed)
    assert (s["mode"] != 0).any() and (s["mode"] == 0).any()


def test_uniform_200_100_reproduces_the_plain_front_given_that_pair(a1):
    B, T = 128, 26
    tp = a1.default_tick_params(0, a1.TICK_MPC)
    tp.gait.horizon = 10
    tp.gait.counter_per_gait, tp.gait.counter_per_swing = 200.0, 100.0
    gait = np.ascontiguousarray(np.repeat(np.array([0.0, 120.0, 120.0, 0.0, 200.0, 100.0])[:, None], B, axis=1))
    run_fronts(a1, tp, gait, B, T, 10, 31)


def test_mixed_gaits_twin_equals_staged(a1):
    """the five gaits in one batch: the fused twin against the staged gait kernels (no plain counterpart)"""
    B, T = 160, 26
    tp = a1.default_tick_params(0, a1.TICK_MPC)
    tp.gait.horizon = 10
    speed = np.ascontiguousarray(np.repeat(np.random.default_rng(3).uniform(1.5, 4.5, B)[None, :], 4, axis=0))
    run_fronts(a1, tp, rows_of(np.arange(B) % 5 + 1), B, T, 10, 41, speed, kinds=(EG.TWIN, EG.STAGED))


def load_swing_golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "swing_v1.npz")) as z:
        return {k: z[k] for k in z.files}


def test_staged_gait_kernels_with_trot_rows_on_the_recorded_ticks(a1):
    G = load_swing_golden()
    R, T = G["contacts"].shape
    gp = a1.default_tick_params(0, a1.TICK_MPC).gait
    gp.horizon = 10
    gait = rows_of([1] * R)
    g = lambda k, t: np.ascontiguousarray(G[k][:, t].T)
    sw = [np.zeros((EG.swing_fields(), R)) for _ in range(2)]
    gcs = [np.zeros((4, R)) for _ in range(2)]
    for t in range(T):
        outs = []
        for side, rows in enumerate((None, gait)):
            mode = np.ascontiguousarray(G["movement_mode"][:, t].astype(np.uint32))
            plan, sched = np.zeros(R, np.uint32), np.zeros((10, R), np.uint32)
            tr, ta, tw = np.zeros((12, R)), np.zeros((12, R)), np.zeros((12, R))
            EG.update_plan(gp, rows, gcs[side], np.ascontiguousarray(G["gait_counter_speed"].T), mode, g("lin_vel", t), g("lin_vel_d", t), g("rot_z", t), g("rot", t),
                           g("root_pos", t), plan, sched, tr, ta, tw)
            fk, con, cur, rc = np.zeros((12, R)), np.zeros(R, np.uint32), np.zeros((12, R)), np.zeros((12, R))
            EG.swing_legs(gp, G["kp"][0], G["kd"][0], DT, rows, sw[side], g("gait_counter", t), np.ascontiguousarray(G["plan_contacts"][:, t]),
                          g("rot_z", t), g("foot_pos_abs", t), g("foot_pos_target_rel", t), g("foot_force", t), fk, con, cur, rc)
            outs.append((gcs[side].copy(), plan, sched, tr, ta, tw, fk, con, cur, rc, sw[side].copy()))
        for a, b in zip(*outs):
            assert a.tobytes() == b.tobytes(), t


def restate_plan(gait, gc, speed, walk, N):
    """the generalised update_plan in numpy: counters, planned mask, schedule rows 0 .. N-1"""
    cpg, cps = gait[4], gait[5]
    c = np.where(walk[None, :], np.fmod(gc + speed, cpg[None, :]), gait[:4])
    plan = np.where(walk[None, :], c <= cps[None, :], True)
    sched = np.zeros((N, gc.shape[1]), np.uint32)
    for st in range(N):
        ci = np.fmod(c + st * speed, cpg[None, :])
        m = np.where(walk[None, :], ci <= cps[None, :], True)
        sched[st] = (m * (1 << np.arange(4))[:, None]).sum(axis=0)
    return c, (plan * (1 << np.arange(4))[:, None]).sum(axis=0).astype(np.uint32), sched


def test_mixed_gaits_match_the_restatement(a1):
    B, T, N = 500, 200, 10
    gp = a1.default_tick_params(0, a1.TICK_MPC).gait
    gp.horizon = N
    gait = rows_of(np.arange(B) % 5 + 1)
    rng = np.random.default_rng(9)
    speed = np.ascontiguousarray(np.repeat(rng.uniform(1.5, 4.5, B)[None, :], 4, axis=0))
    speed[:, ::7] = 2.0
    gc, ref = np.zeros((4, B)), np.zeros((4, B))
    for t in range(T):
        walk = (t % 60 >= 3) & (rng.random(B) < 0.98)
        plan, sched = np.zeros(B, np.uint32), np.zeros((N, B), np.uint32)
        EG.update_plan(gp, gait, gc, speed, walk.astype(np.uint32), None, None, None, None, None, plan, sched, None, None, None)
        c, p, s = restate_plan(gait, ref, speed, walk, N)
        ref = c
        assert np.array_equal(gc, c) and np.array_equal(plan, p) and np.array_equal(sched, s), t


def cycle_masks(gtype, speed=2.0):
    """planned masks over one cycle at equal leg speeds, from a standstill tick (offsets) into walking"""
    gp_row = rows_of([gtype])
    B = 1
    import a1mpc
    gp = a1mpc.default_tick_params(0, a1mpc.TICK_MPC).gait
    gc = np.zeros((4, B))
    sp = np.full((4, B), speed)
    masks = []
    for t in range(1 + int(gp_row[4, 0] / speed)):
        plan = np.zeros(B, np.uint32)
        EG.update_plan(gp, gp_row, gc, sp, np.array([1 if t else 0], np.uint32), None, None, None, None, None, plan, None, None, None, None)
        if t:
            masks.append(int(plan[0]))
    return masks


def _legs(m):
    return [(m >> i) & 1 for i in range(4)]   # FL FR RL RR


def test_contact_patterns_over_a_cycle(a1):
    trot, pace, bound, pronk, walk = (cycle_masks(g) for g in (1, 2, 3, 4, 5))
    for m in trot:
        fl, fr, rl, rr = _legs(m)
        assert fl == rr and fr == rl
    for m in pace:
        fl, fr, rl, rr = _legs(m)
        assert fl == rl and fr == rr
    for m in bound:
        fl, fr, rl, rr = _legs(m)
        assert fl == fr and rl == rr
    for masks in (trot, pace, bound):
        assert set(bin(m).count("1") for m in masks) <= {2, 4} and any(bin(m).count("1") == 2 for m in masks)
    assert set(pronk) == {0, 15}
    assert min(bin(m).count("1") for m in walk) >= 3
    # each leg swings exactly once per cycle, and the swings start in the order RL, FL, RR, FR
    starts = []
    for i in range(4):
        down = [(m >> i) & 1 for m in walk]
        lifts = [t for t in range(len(down)) if down[t] == 0 and down[t - 1] == 1]
        assert len(lifts) == 1, (i, down)
        starts.append(lifts[0])
    assert [ {0: "FL", 1: "FR", 2: "RL", 3: "RR"}[i] for i in np.argsort(starts)] == ["RL", "FL", "RR", "FR"]


def test_row_check_rules(a1):
    B = 300
    good = rows_of(np.arange(B) % 5 + 1)
    assert EG.check(good) is None
    cases = [(7, 4, np.nan, 1), (9, 0, np.inf, 1), (11, 5, 0.0, 2), (13, 5, 240.0, 2), (15, 5, -1.0, 2), (17, 2, 240.0, 3), (19, 3, -0.5, 3),
             (21, 4, 100.0, 3)]   # cpg 100 < offset 120 of a trot row: cps 120 >= cpg breaks rule 2 first
    for b, k, v, rule in cases:
        g = good.copy()
        g[k, b] = v
        want = 2 if (b, k, v) == (21, 4, 100.0) else rule
        assert EG.check(g) == (b, want), (b, k, v)
    g = good.copy()
    g[5, 250] = 0.0
    g[0, 40] = 240.0
    assert EG.check(g) == (40, 3)      # the first bad robot


def test_gait_row_table(a1):
    for t, row in TABLE.items():
        assert np.array_equal(a1.gait_row(t), np.array(row, dtype=np.float64)), t
    for bad in (0, 6, -1):
        with pytest.raises(a1.A1MpcError, match="unknown gait type"):
            a1.gait_row(bad)
    assert (a1.GAIT_TROT, a1.GAIT_PACE, a1.GAIT_BOUND, a1.GAIT_PRONK, a1.GAIT_WALK) == (1, 2, 3, 4, 5)
    for t in TABLE:
        assert EG.check(rows_of([t])) is None
