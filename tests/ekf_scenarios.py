"""Walking sensor streams for the batched Kalman filter (a1mpc_ekf_update_batch), and the two checks that run on them against the
oracle: a long run, each side carrying its own filter state from tick to tick, and the NUMERICAL contract for non-finite inputs.  The
GPU tests (test_gpu_ekf.py) and the emulator tests (test_emu_ekf.py) call both through a backend with the methods

    kin(q, dq, rot) -> foot_pos_rel [12,B], foot_vel_rel [12,B]         the device's leg kinematics
    init(foot_pos_rel, rot) -> handle                                  a fresh filter state of B robots
    update(handle, flat, inp, fpr, fvr, tick) -> pos, vel, ec, status  one a1mpc_ekf_update_batch
    state(handle) -> [B,342] float64                                   x[18], P[18,18] per robot, as the device holds them
    clone(handle) -> handle                                            a second filter state with the same bytes
"""
import numpy as np

from oracle import ekf_batch_oracle_py as OB

DT = 0.0025
Q0 = np.array([0.0, 0.8, -1.6] * 4)
# GazeboA1ROS.cpp:76-97 (ox, oy, d, lt, lc per leg)
RHO_FIX = np.array([[0.1805, 0.047, 0.0838, 0.21, 0.21], [0.1805, -0.047, -0.0838, 0.21, 0.21],
                    [-0.1805, 0.047, 0.0838, 0.21, 0.21], [-0.1805, -0.047, -0.0838, 0.21, 0.21]])
RHO_OPT = np.zeros((4, 3))
# the two legs of each diagonal (trot) or each end (bound) move together
GAIT_PAIRS = {"trot": (0, 1, 1, 0), "bound": (0, 0, 1, 1)}
STATUS_OPTIMAL, STATUS_NUMERICAL = 0, 3


def rot_rpy(r, p, y):
    """[9,B] row-major R = Rz(y) Ry(p) Rx(r) of B angle triples"""
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    return np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
                     sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
                     -sp, cp * sr, cp * cr])


class WalkStream:
    """Seeded sensor stream of B robots.  step() returns one tick's inputs: movement_mode [B], acc [3,B], gyro [3,B], rot [9,B],
    joint_pos / joint_vel [12,B] and foot_force [4,B].

    * Joint angles random-walk around (0, 0.8, -1.6) per leg, pulled back by a spring; joint_vel is the rate the next angle is
      integrated with (q' = q + dt dq), so the two match.
    * Each robot trots or bounds (GAIT_PAIRS) with its own period (160-240 ticks, half of it stance) and phase.  Foot force: stance
      40-140 N, swing -5-20 N; 2 % of the readings are exactly 0 N and 2 % exactly 100 N, the ends of the contact clamp.
    * Mode: standstill for the first 20-80 ticks, then walking segments of 300-900 ticks and standstill segments of 30-150 ticks
      alternate, each robot on its own clock.  Standing robots load all four feet.
    * IMU: acc = R' (0, 0, 9.81) + N(0, 0.3), gyro = the yaw rate plus N(0, 0.05); roll and pitch wander by a few hundredths of a
      radian and the yaw turns at a slowly changing rate of up to about 0.3 rad/s."""

    def __init__(self, B, seed, gaits=("trot", "bound")):
        self.B = B
        self.rng = rng = np.random.default_rng(seed)
        self.q = np.tile(Q0[:, None], (1, B)) + rng.normal(0, 0.1, (12, B))
        self.dq = rng.normal(0, 0.5, (12, B))
        self.pair = np.array([GAIT_PAIRS[gaits[i]] for i in rng.integers(0, len(gaits), B)]).T   # [4,B]
        self.period = rng.choice([160, 200, 240], B)
        self.phase = rng.integers(0, 240, B)
        self.mode = np.zeros(B, dtype=np.uint32)
        self.next_toggle = rng.integers(20, 81, B)
        self.rpy = np.stack([rng.normal(0, 0.03, B), rng.normal(0, 0.03, B), rng.uniform(-np.pi, np.pi, B)])
        self.yaw_rate = rng.uniform(-0.3, 0.3, B)
        self.t = 0

    def step(self):
        rng, B, t = self.rng, self.B, self.t
        flip = t >= self.next_toggle
        if flip.any():
            self.mode[flip] ^= 1
            walk = self.mode[flip] == 1
            self.next_toggle[flip] = t + np.where(walk, rng.integers(300, 901, flip.sum()), rng.integers(30, 151, flip.sum()))
        walking = self.mode == 1
        # joints: a damped spring about Q0 driven by noise; the returned angle is integrated with the returned rate
        q, dq = self.q, self.dq
        self.q = q + DT * dq
        self.dq = dq + DT * (-40.0 * (q - Q0[:, None]) - 8.0 * dq) + np.where(walking, 0.3, 0.1) * rng.standard_normal((12, B))
        # gait schedule: pair 0 in stance for the first half of the period, pair 1 for the second
        first_half = ((self.phase + t) % self.period) < self.period // 2
        stance = (self.pair == 0) == first_half[None, :]
        stance |= ~walking[None, :]
        force = np.where(stance, rng.uniform(40.0, 140.0, (4, B)), rng.uniform(-5.0, 20.0, (4, B)))
        u = rng.random((4, B))
        force[u < 0.02] = 0.0
        force[(u >= 0.02) & (u < 0.04)] = 100.0
        # orientation and IMU
        self.yaw_rate = np.clip(self.yaw_rate + rng.normal(0, 0.01, B), -0.3, 0.3)
        self.rpy[:2] += -0.01 * self.rpy[:2] + rng.normal(0, 0.003, (2, B))
        self.rpy[2] += DT * self.yaw_rate
        rot = rot_rpy(*self.rpy)
        R = rot.reshape(3, 3, B)
        acc = 9.81 * R[2] + rng.normal(0, 0.3, (3, B))          # R' (0, 0, 9.81) = 9.81 x the third row of R
        gyro = rng.normal(0, 0.05, (3, B)); gyro[2] += self.yaw_rate
        self.t += 1
        return dict(mode=self.mode.copy(), acc=acc, gyro=gyro, rot=np.ascontiguousarray(rot), joint_pos=q, joint_vel=dq, force=force)


def oracle_threads(O):
    return max(1, O.effective_cores()[0])


def oracle_init(O, fpr, rot):
    """[B,342]: oracle_ekf_init of every robot"""
    return np.stack([np.concatenate([x, P.ravel()]) for x, P in (O.ekf_init(fpr[:, b], rot[:, b]) for b in range(fpr.shape[1]))])


def cut_rows(state):
    """[B] bool: the position-drift cut (A1BasicEKF.cpp:144-148) left P[0, 2:] exactly zero"""
    return (state[:, 18 + 2:18 + 18] == 0.0).all(axis=1)


def compare(state, outs, ostate, oouts, rows=slice(None)):
    """worst |device - oracle| over x, P, root_pos and root_lin_vel of the robots `rows`; asserts the contact masks agree"""
    pos, vel, ec, status = outs
    opos, ovel, oec, orc = oouts
    assert (status[rows] == STATUS_OPTIMAL).all() and (orc[rows] == 0).all(), (np.unique(status[rows]), np.unique(orc[rows]))
    assert (ec[rows] == oec[rows]).all(), np.nonzero(ec[rows] != oec[rows])
    return max(float(np.abs(state[rows] - ostate[rows]).max()), float(np.abs(pos[:, rows] - opos[:, rows]).max()),
               float(np.abs(vel[:, rows] - ovel[:, rows]).max()))


def walk_against_oracle(dev, O, B, T, flat, seed, tol=1e-10):
    """T ticks of a WalkStream of B robots through the backend and the oracle, each carrying its own state.  Every tick: x, P, root_pos,
    root_lin_vel within tol, the contact masks equal, status 0, and the cut decision (cut_rows) equal on every robot.  Returns the worst
    difference and the [T,B] bool cut record of the device."""
    ws = WalkStream(B, seed)
    nt = oracle_threads(O)
    inp = ws.step()
    fpr, fvr = dev.kin(inp["joint_pos"], inp["joint_vel"], inp["rot"])
    h = dev.init(fpr, inp["rot"])
    ost = oracle_init(O, fpr, inp["rot"])
    worst = float(np.abs(dev.state(h) - ost).max())
    cuts = np.zeros((T, B), dtype=bool)
    for t in range(T):
        inp = ws.step()
        fpr, fvr = dev.kin(inp["joint_pos"], inp["joint_vel"], inp["rot"])
        outs = dev.update(h, flat, inp, fpr, fvr, t)
        oouts = OB.ekf_update_batch(ost, DT, flat, inp["mode"], inp["acc"], inp["gyro"], inp["rot"], fpr, fvr, inp["force"], nthreads=nt)
        st = dev.state(h)
        w = compare(st, outs, ost, oouts)
        assert w <= tol, (t, w)
        worst = max(worst, w)
        cuts[t] = cut_rows(st)
        oc = cut_rows(ost)
        assert (cuts[t] == oc).all(), (t, np.nonzero(cuts[t] != oc)[0][:10])
    return worst, cuts


# ---------------------------------------------------------------------------------------------------------------------------------
# NUMERICAL contract.  A poison plan puts one non-finite value into one input of chosen robots:
#   kind          input, row               value             mode forced   expected
#   acc           imu_acc, 0-2             NaN / +Inf / -Inf  -             NUMERICAL
#   gyro          imu_ang_vel, 0-2         NaN / +Inf / -Inf  -             NUMERICAL
#   rot           rot, 0-8                 NaN / +Inf / -Inf  -             NUMERICAL
#   fpr           foot_pos_rel, 0-11       NaN / +Inf / -Inf  -             NUMERICAL
#   fvr           foot_vel_rel, 0-11       NaN / +Inf / -Inf  -             NUMERICAL
#   force_nan     foot_force, 0-3          NaN                walking       NUMERICAL, that leg's contact bit 1
#   force_inf     foot_force, 0-3          +Inf / -Inf        walking       updated: the clamp gives contact 1 / 0
#   force_stand   foot_force, 0-3          NaN / +Inf / -Inf  standstill    updated: standstill ignores the force
# ---------------------------------------------------------------------------------------------------------------------------------
KINDS = {"acc": ("acc", 3), "gyro": ("gyro", 3), "rot": ("rot", 9), "fpr": ("fpr", 12), "fvr": ("fvr", 12),
         "force_nan": ("force", 4), "force_inf": ("force", 4), "force_stand": ("force", 4)}
NUMERICAL_KINDS = ("acc", "gyro", "rot", "fpr", "fvr", "force_nan")


def poison_plan(B, per_kind, rng):
    """[(kind, robot, row, value)]: per_kind distinct robots for each kind"""
    robots = rng.permutation(B)[:per_kind * len(KINDS)]
    plan = []
    for k, kind in enumerate(KINDS):
        _, rows = KINDS[kind]
        for j, b in enumerate(robots[k * per_kind:(k + 1) * per_kind]):
            if kind == "force_nan":
                v = np.nan
            elif kind == "force_inf":
                v = (np.inf, -np.inf)[j % 2]
            else:
                v = (np.nan, np.inf, -np.inf)[j % 3]
            plan.append((kind, int(b), int(rng.integers(0, rows)), v))
    return plan


def apply_poison(inp, fpr, fvr, plan):
    """copies of (inputs, fpr, fvr) with the plan's values in place and the modes it forces"""
    inp = {k: v.copy() for k, v in inp.items()}
    arrs = dict(inp, fpr=fpr.copy(), fvr=fvr.copy())
    for kind, b, row, v in plan:
        arrs[KINDS[kind][0]][row, b] = v
        if kind in ("force_nan", "force_inf"):
            arrs["mode"][b] = 1
        elif kind == "force_stand":
            arrs["mode"][b] = 0
    return {k: arrs[k] for k in inp}, arrs["fpr"], arrs["fvr"]


def contact_bits(mode, force):
    """the estimated-contact masks of A1BasicEKF.cpp:78-86 and :157-160, with the reference's comparisons: NaN force -> bit 1"""
    r = force / 100.0
    with np.errstate(invalid="ignore"):
        ec = np.where(r < 0, 0.0, np.where(1 < r, 1.0, r))
        ec = np.where(mode[None, :] == 0, 1.0, ec)
        bit = ~(ec < 0.5)
    return (bit * (1 << np.arange(4))[:, None]).sum(axis=0).astype(np.uint32)


def numerical_contract(dev, O, B, flat, seed, warm_ticks, per_kind, next_ticks=2, tol=1e-10):
    """warm_ticks finite ticks, then one tick with the poison plan, then next_ticks finite ticks, on two filter states that start from
    the same bytes: h gets the poisoned tick, its clone u the same tick without the poison.  Checks:
      * every robot of a NUMERICAL kind: status NUMERICAL, state bytes as before the tick, root_pos / root_lin_vel bit-equal to that
        state's x[0:3] / x[3:6], contact bits by contact_bits on the poisoned inputs;
      * every robot of the other two kinds: updated, status 0, within tol of the oracle run on the poisoned inputs;
      * every robot without poison: state and every output bit-identical to u's;
      * the following finite ticks: every robot of h within tol of the oracle, whose NUMERICAL robots kept their state too.
    Returns the plan and the worst difference against the oracle."""
    ws = WalkStream(B, seed)
    rng = np.random.default_rng(seed + 1)
    nt = oracle_threads(O)
    inp = ws.step()
    fpr, fvr = dev.kin(inp["joint_pos"], inp["joint_vel"], inp["rot"])
    h = dev.init(fpr, inp["rot"])
    ost = oracle_init(O, fpr, inp["rot"])
    worst = float(np.abs(dev.state(h) - ost).max())
    tick = 0

    def finite_tick(handle):
        nonlocal worst, tick
        inp = ws.step()
        fpr, fvr = dev.kin(inp["joint_pos"], inp["joint_vel"], inp["rot"])
        outs = dev.update(handle, flat, inp, fpr, fvr, tick)
        oouts = OB.ekf_update_batch(ost, DT, flat, inp["mode"], inp["acc"], inp["gyro"], inp["rot"], fpr, fvr, inp["force"], nthreads=nt)
        w = compare(dev.state(handle), outs, ost, oouts)
        assert w <= tol, (tick, w)
        worst = max(worst, w)
        tick += 1

    for _ in range(warm_ticks):
        finite_tick(h)
    u = dev.clone(h)
    before = dev.state(h).copy()
    assert before.tobytes() == dev.state(u).tobytes()

    plan = poison_plan(B, per_kind, rng)
    inp = ws.step()
    fpr, fvr = dev.kin(inp["joint_pos"], inp["joint_vel"], inp["rot"])
    pinp, pfpr, pfvr = apply_poison(inp, fpr, fvr, plan)
    # U runs the poisoned robots' forced modes too, so that only the non-finite values differ between the two calls
    uinp = dict(inp, mode=pinp["mode"])
    pos, vel, ec, status = dev.update(h, flat, pinp, pfpr, pfvr, tick)
    upos, uvel, uec, ustatus = dev.update(u, flat, uinp, fpr, fvr, tick)
    tick += 1
    after, uafter = dev.state(h), dev.state(u)

    numerical = np.zeros(B, dtype=bool)
    poisoned = np.zeros(B, dtype=bool)
    for kind, b, row, v in plan:
        poisoned[b] = True
        numerical[b] = kind in NUMERICAL_KINDS
    # the poisoned robots
    nb = np.nonzero(numerical)[0]
    assert (status[nb] == STATUS_NUMERICAL).all(), [(k, b, row, v, int(status[b])) for k, b, row, v in plan if numerical[b] and status[b] != STATUS_NUMERICAL]
    assert after[nb].tobytes() == before[nb].tobytes()
    assert pos[:, nb].tobytes() == np.ascontiguousarray(before[nb, 0:3].T).tobytes()
    assert vel[:, nb].tobytes() == np.ascontiguousarray(before[nb, 3:6].T).tobytes()
    assert (ec == contact_bits(pinp["mode"], pinp["force"])).all()
    for kind, b, row, v in plan:
        if kind == "force_nan":
            assert (int(ec[b]) >> row) & 1 == 1
    # the oracle on the poisoned inputs: its NaN-force robots end NUMERICAL too; the robots the device reports NUMERICAL keep their state
    ost_before = ost.copy()
    oouts = OB.ekf_update_batch(ost, DT, flat, pinp["mode"], pinp["acc"], pinp["gyro"], pinp["rot"], pfpr, pfvr, pinp["force"], nthreads=nt)
    for kind, b, row, v in plan:
        if kind == "force_nan":
            assert oouts[3][b] == STATUS_NUMERICAL, (b, oouts[3][b])
    ost[nb] = ost_before[nb]
    rest = np.nonzero(~numerical)[0]
    w = compare(after, (pos, vel, ec, status), ost, oouts, rows=rest)
    assert w <= tol, w
    worst = max(worst, w)
    # every robot without poison: the same bytes as the call without the poison
    cl = np.nonzero(~poisoned)[0]
    assert after[cl].tobytes() == uafter[cl].tobytes()
    for a, b in ((pos, upos), (vel, uvel)):
        assert a[:, cl].tobytes() == b[:, cl].tobytes()
    assert ec[cl].tobytes() == uec[cl].tobytes() and status[cl].tobytes() == ustatus[cl].tobytes()
    # the next finite ticks continue from the untouched state
    for _ in range(next_ticks):
        finite_tick(h)
    return plan, worst
