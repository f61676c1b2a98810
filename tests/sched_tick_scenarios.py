"""Scheduled MPC solves as a closed-loop control tick poses them, for tests/test_emu_sched_tick.py (CPU emulator) and
tests/test_gpu_sched_tick.py (C ABI).

tick_solve_inputs runs the oracle chain of tests/test_gpu_command.py's MPC closed loop on the CPU (orientation, leg kinematics,
command, update_plan with its per-step schedule, swing legs, EKF, terrain pitch) and keeps every tick's solve inputs.  The chain
runs on the CPU for every consumer: the device chain matches it only to 1e-8 in x0, and a QP near a degenerate face must be the
same QP on the emulator, on the GPU and in a fixture.

The run is long enough to reach the schedules update_plan makes in a walking robot, which a short run or a1mpc_gen_schedule
never poses:
  * standstill (ticks 0-4): all four feet in every step, counters reset to 0 / 120;
  * half of the robots walk from tick 5 to the end.  update_plan's step st is c + st * speed with c = j * speed on the j-th
    walking tick, so with counter_per_swing = 120 a horizon window holds a four-foot crossing step once j + 9 reaches a multiple
    of 120 / speed: from tick 25 (speed 4), 35 (speed 3) and 55 (speed 2);
  * a quarter leaves walking at tick 18 and comes back at tick 24, the last quarter leaves at 18 and comes back at 34: counters
    restart, phases stay locked, and the warm start sees a walk / stand switch;
  * the swing stage's early contacts (foot forces are uniform in 0-80 N).
Deterministic: numpy, seeded.

Three schedule variants per tick (variant()):
  plan     update_plan's schedule as it comes;
  early    step 0 replaced by the swing stage's contacts (plan OR early contact), what a controller that honours an early touchdown
           poses: adds three-foot steps;
  terrain  the plan schedule with each foot's normal tilted by the tick's terrain pitch ref[1] about the yaw frame's y axis,
           n = Rz(yaw) Ry(pitch) e_z (r stays isotropic, as normals require)."""
import numpy as np

from command_scenarios import DT, HMAX, HMIN, KP_LINEAR, KP_LOCK
from common import estimation_scenario
from swing_scenarios import CPS, KD_ROS, KP_ROS
from tick_scenarios import tick_inputs

VARIANTS = ("plan", "early", "terrain")


def _toggles(B, T):
    """cmd[:, 6]: walk from tick 5; [0, B/4) out at 18 and in at 24, [B/4, B/2) out at 18 and in at 34, [B/2, B) walk throughout"""
    tog = np.zeros((T, B))
    for t, lo, hi in ((5, 0, B), (18, 0, B // 2), (24, 0, B // 4), (34, B // 4, B // 2)):
        if t < T:
            tog[t, lo:hi] = 1.0
    return tog


def tick_solve_inputs(B, T, seed, N=10):
    """the oracle chain over T ticks of B robots; returns dict of per-tick arrays
       x0 [T,12,B], rot [T,9,B], foot [T,12,B], ref [T,9,B]  the solve's inputs (foot = foot_pos_abs)
       contact [T,B]   the swing stage's contacts (plan OR early contact)
       plan [T,B]      update_plan's planned contacts
       sched [T,N,B]   update_plan's per-step schedule
       mode [T,B]      movement_mode
       fk [T,12,B], jac [T,36,B]  the swing stage's forces and the leg Jacobians (robot-major 4 x 3 x 3), for joint torques
    and seqs (the tick inputs of tick_scenarios.tick_inputs with this run's toggles), speed [4,B], rho_opt [12], rho_fix [20], seed."""
    import a1mpc
    from oracle import command_oracle_py as CO
    from oracle import oracle_py as O
    from oracle import swing_oracle_py as SO
    seqs, speed = tick_inputs(B, T, seed)
    seqs["cmd"][:, 6] = _toggles(B, T)
    quat, gyro, acc, q, dq, force, cmd = (seqs[k] for k in ("quat", "gyro", "acc", "joint_pos", "joint_vel", "foot_force", "cmd"))
    _, rho_opt, rho_fix, _, _, _ = estimation_scenario(4, 5)
    rho_opt, rho_fix = rho_opt.reshape(12), rho_fix.reshape(20)
    gp = a1mpc.default_gait_params(N)
    cp = a1mpc.default_command_params(a1mpc.VARIANT_GAZEBO)
    ori, com, sw = CO.Orientation(B), CO.Command(B, 0, cp.body_height, HMIN, HMAX, KP_LINEAR, KP_LOCK), SO.Swing(B)
    x0 = np.zeros((12, B)); gc = np.zeros((4, B)); row1 = np.zeros(B)
    xs, Ps = [None] * B, [None] * B
    keys = dict(x0=((12,), np.float64), rot=((9,), np.float64), foot=((12,), np.float64), ref=((9,), np.float64), contact=((), np.uint32),
                plan=((), np.uint32), sched=((N,), np.uint32), mode=((), np.uint32), fk=((12,), np.float64), jac=((36,), np.float64))
    out = {k: np.zeros((T,) + s + (B,), dtype=dt) for k, (s, dt) in keys.items()}
    for t in range(T):
        o = ori(quat[t], gyro[t], acc[t])
        x0[0:3], x0[6:9] = o["euler"], o["ang_vel"]
        R = o["rot"].T.reshape(B, 3, 3)
        p = np.zeros((B, 4, 3)); J = np.zeros((B, 4, 3, 3))
        for b in range(B):
            for leg in range(4):
                p[b, leg], J[b, leg] = O.leg_kinematics(q[t, 3 * leg:3 * leg + 3, b], rho_opt[3 * leg:3 * leg + 3], rho_fix[5 * leg:5 * leg + 5])
        fpr = p.reshape(B, 12).T.copy()
        fvr = np.stack([np.einsum("bij,jb->ib", J[:, leg], dq[t, 3 * leg:3 * leg + 3]) for leg in range(4)]).reshape(12, B)
        fabs = np.einsum("bij,blj->bli", R, p).reshape(B, 12).T.copy()
        mode, _, ref, _ = com(DT, cmd[t], x0[3:6], row1)
        plan = np.zeros(B, dtype=np.uint32); sched = np.zeros((N, B), dtype=np.uint32); trel = np.zeros((12, B))
        for b in range(B):
            gc[:, b], plan[b], sched[:, b], trel[:, b], _, _ = O.update_plan(gp, mode[b], gc[:, b], speed[:, b], x0[9:12, b], ref[5:8, b],
                                                                             o["rot_z"][:, b], o["rot"][:, b], x0[3:6, b])
        fk, con, _, _ = sw.legs(CPS, DT, KP_ROS, KD_ROS, gc, plan, o["rot_z"], fabs, trel, force[t])
        for b in range(B):
            if t == 0:
                xs[b], Ps[b] = O.ekf_init(fpr[:, b], o["rot"][:, b])
            else:
                xs[b], Ps[b], x0[3:6, b], x0[9:12, b], _, rc = O.ekf_update(xs[b], Ps[b], DT, 1, mode[b], o["imu_acc"][:, b], o["imu_ang_vel"][:, b],
                                                                            o["rot"][:, b], fpr[:, b], fvr[:, b], force[t, :, b])
                assert rc == 0, (t, b)
        sw.terrain(1, x0[3:6], ref)
        row1 = ref[1].copy()
        for k, v in dict(x0=x0, rot=o["rot"], foot=fabs, ref=ref, contact=con, plan=plan, sched=sched, mode=mode, fk=fk,
                         jac=J.reshape(B, 36).T).items():
            out[k][t] = v
    out.update(seqs=seqs, speed=speed, rho_opt=rho_opt, rho_fix=rho_fix, seed=seed)
    return out


def normals_of(rot, pitch):
    """[12,B] per-foot normals Rz(yaw) Ry(pitch) e_z, all four feet alike; yaw from the body rotation rot [9,B] (row-major)"""
    yaw = np.arctan2(rot[3], rot[0])
    n = np.stack([np.cos(yaw) * np.sin(pitch), np.sin(yaw) * np.sin(pitch), np.cos(pitch)])
    return np.ascontiguousarray(np.tile(n, (4, 1)))


def variant(d, name, t):
    """tick t of variant `name`: (state dict with contact = step 0 of the schedule, sched [N,B], normals [12,B] or None)"""
    sched = d["sched"][t].copy()
    if name == "early":
        sched[0] = d["contact"][t]
    normals = normals_of(d["rot"][t], d["ref"][t][1]) if name == "terrain" else None
    st = {k: np.ascontiguousarray(d[k][t]) for k in ("x0", "rot", "foot", "ref")}
    st["contact"] = np.ascontiguousarray(sched[0])
    return st, np.ascontiguousarray(sched), normals


def stacked(d, name, ticks=None):
    """the QPs of the given ticks (all by default) of variant `name` as one batch, tick-major (column t * B + b): the cold solves
    of different ticks are independent, and one large call keeps every worker of the emulator and every SM busy"""
    parts = [variant(d, name, t) for t in (range(d["sched"].shape[0]) if ticks is None else ticks)]
    st = {k: np.ascontiguousarray(np.concatenate([p[0][k] for p in parts], axis=-1)) for k in parts[0][0]}
    sched = np.ascontiguousarray(np.concatenate([p[1] for p in parts], axis=1))
    normals = np.ascontiguousarray(np.concatenate([p[2] for p in parts], axis=1)) if parts[0][2] is not None else None
    return st, sched, normals


def _popcount(m):
    m = np.asarray(m, dtype=np.uint32)
    return ((m >> 0) & 1) + ((m >> 1) & 1) + ((m >> 2) & 1) + ((m >> 3) & 1)


def two_feet(sched):
    """[B] bool: every step of the schedule [N,B] has exactly two stance feet (the robots pack_ext2_kernel sends to the compacted
    kernel)"""
    return (_popcount(sched) == 2).all(axis=0)


def sched_census(d, name):
    """counts over every (tick, robot) of variant `name`: robots routed to the compacted and to the general kernel; schedules with a
    step of four, three or zero stance feet (zero: with contact elsewhere in the horizon); all-four standstill schedules; windows
    posed right after a walk / stand switch (the stored warm faces belong to the other mode); robots with an early contact"""
    T = d["sched"].shape[0]
    c = dict(QPs=0, compact=0, general=0, four=0, three=0, zero=0, standstill=0, switch=0, early=0)
    for t in range(T):
        _, sched, _ = variant(d, name, t)
        pc = _popcount(sched)
        some = (sched != 0).any(axis=0)
        two = two_feet(sched)
        c["QPs"] += sched.shape[1]
        c["compact"] += int(two.sum())
        c["general"] += int((~two & some).sum())
        c["four"] += int(((pc == 4).any(axis=0) & (d["mode"][t] != 0)).sum())   # walking: a crossing step, or both swing feet down early
        c["three"] += int((pc == 3).any(axis=0).sum())
        c["zero"] += int(((pc == 0).any(axis=0) & some).sum())
        c["standstill"] += int((sched == 15).all(axis=0).sum())
        if t > 0:
            c["switch"] += int((d["mode"][t] != d["mode"][t - 1]).sum())
        c["early"] += int((d["contact"][t] & ~d["plan"][t] != 0).sum())
    return c


def _to_terrain(u, normals):
    """u_full [B,12N] world frame -> each foot's terrain frame, R' f with R the Rodrigues rotation z -> n (the frame in which the
    solver's pyramid is axis aligned)"""
    B = u.shape[0]
    n = normals.T.reshape(B, 4, 3)
    n = n / np.linalg.norm(n, axis=2, keepdims=True)
    v = np.stack([-n[..., 1], n[..., 0], np.zeros_like(n[..., 0])], axis=-1)         # e_z x n
    K = np.zeros((B, 4, 3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 0], K[..., 1, 2], K[..., 2, 0], K[..., 2, 1] = -v[..., 2], v[..., 1], v[..., 2], -v[..., 0], -v[..., 1], v[..., 0]
    R = np.eye(3) + K + np.einsum("blij,bljk->blik", K, K) / (1.0 + n[..., 2])[..., None, None]
    f = u.reshape(B, -1, 4, 3)
    return np.einsum("blji,bslj->bsli", R, f).reshape(B, -1)


def face_census(d, name, u):
    """envelope_scenarios.census of the oracle's optimum u_full [T*B,12N] of stacked(d, name); with the terrain variant's normals the
    faces are those of each foot's terrain-frame pyramid"""
    from envelope_scenarios import census
    _, sched, normals = stacked(d, name)
    return census(u if normals is None else _to_terrain(u, normals), None, sched=sched)


def check_floors(tag, c, floors):
    """prints the census and asserts each floor (a count): a later edit of the generator cannot make the family easy"""
    print("census %-8s %s" % (tag, "  ".join("%s %d" % kv for kv in c.items())))
    for k, v in floors.items():
        assert c[k] >= v, (tag, k, c[k], v)


def describe(d, name, qps):
    """the inputs of QPs `qps` (columns t * B + b of stacked(d, name)) with their seed, variant, tick and robot, for a failure
    message that can become a fixture without a rerun"""
    B = d["sched"].shape[2]
    lines = ["seed %d, variant %s" % (d["seed"], name)]
    for i in np.atleast_1d(qps)[:8]:
        t, b = divmod(int(i), B)
        st, sc, nm = variant(d, name, t)
        lines.append("tick %d robot %d: x0 %s rot %s foot %s ref %s sched %s%s" % (
            t, b, st["x0"][:, b].tolist(), st["rot"][:, b].tolist(), st["foot"][:, b].tolist(), st["ref"][:, b].tolist(), sc[:, b].tolist(),
            (" normals %s" % nm[:, b].tolist()) if nm is not None else ""))
    return "\n".join(lines)
