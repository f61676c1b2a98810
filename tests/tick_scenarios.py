"""Inputs of a run of control ticks, and the same run as a hand-built chain of the staged entry points (the chain of
tests/test_gpu_command.py's closed loops), for the tick tests."""
import ctypes as C

import numpy as np

from command_scenarios import command_sequence, imu_sequence


def tick_inputs(B, T, seed):
    """[T][rows][B] arrays of the eight tick inputs, gait_counter_speed [4][B]: standstill, walking from tick 5, half of the robots toggled
    out at tick 18 and a quarter at tick 24 (back in for the half that was out, out for the rest of the quarter)"""
    rng = np.random.default_rng(seed)
    quat, gyro, acc = imu_sequence(B, T, seed, gimbal_share=0.0, gentle=True)
    cmd, _ = command_sequence(B, T, seed + 1)
    cmd[:, 6] = 0.0
    if T > 5:
        cmd[5, 6] = 1.0
    if T > 18:
        cmd[18, 6, : B // 2] = 1.0
    if T > 24:
        cmd[24, 6, : B // 4] = 1.0
    cmd[:, 4] = np.where(np.arange(B) % 2 == 0, 0.3, -0.2)[None, :]
    q = np.tile(np.array([0.0, 0.8, -1.6] * 4)[None, :, None], (T, 1, B)) + 0.05 * rng.standard_normal((T, 12, B))
    dq = 0.5 * rng.standard_normal((T, 12, B))
    force = rng.uniform(0.0, 80.0, (T, 4, B))
    speed = np.ascontiguousarray(np.repeat(rng.choice([2.0, 3.0, 4.0], B)[None, :], 4, axis=0))
    seqs = dict(quat=quat, gyro=gyro, acc=acc, joint_pos=q, joint_vel=dq, foot_force=force, cmd=np.ascontiguousarray(cmd))
    return {k: np.ascontiguousarray(v) for k, v in seqs.items()}, speed


def off(p, nbytes):
    return C.c_void_p((p.value or 0) + nbytes)


def h2d(a1, eng, dst, a):
    a = np.ascontiguousarray(a)
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, dst, a.ctypes.data, a.nbytes))


def d2h(a1, eng, src, shape, dtype=np.float64):
    a = np.zeros(shape, dtype=dtype)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, a.ctypes.data, src, a.nbytes))
    eng.sync()
    return a


class DeviceSeqs:
    """the whole run's inputs on the device; at(name, t) points at tick t"""

    def __init__(self, a1, eng, seqs, speed):
        self.a1, self.eng, self.seqs = a1, eng, seqs
        self.p = {k: eng.dalloc(v.nbytes) for k, v in seqs.items()}
        for k, v in seqs.items():
            h2d(a1, eng, self.p[k], v)
        self.speed = eng.dalloc(speed.nbytes)
        h2d(a1, eng, self.speed, speed)

    def at(self, k, t):
        return off(self.p[k], t * self.seqs[k][0].nbytes)

    def free(self):
        for p in list(self.p.values()) + [self.speed]:
            self.a1.lib().a1mpc_device_free(self.eng.h, p)


OUT_SPECS = dict(tau=((12,), np.float64), f_body=((12,), np.float64), status=((), np.int32), contacts=((), np.uint32),
                 movement_mode=((), np.uint32), x0=((12,), np.float64), ref=((9,), np.float64))


def staged_chain(a1, eng, tp, ds, B, T, dt):
    """the tick's stages as separate entry points on device pointers, from the same start state as a1mpc_tick_create; returns one dict of
    host outputs per tick"""
    L = a1.lib()
    mpc = tp.mode == a1.TICK_MPC
    N = eng.cfg.horizon
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status")}
    filtered = tp.command.variant != a1.VARIANT_HARDWARE
    imu = eng.imu_alloc(B) if filtered else None
    sw, ekf = eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B))
    warm = eng.warm_alloc(B) if N == 10 else None
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    a1._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), dv["ref"] if mpc else None, B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    inp = a1.Inputs(dv["x0"], dv["rot"], dv["foot"], dv["ref"], u["contact"], B)
    out = a1.Outputs(dv["f_body"], u["status"], None, None, B)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    kdl, kpa, kda = arr(tp.kd_linear), arr(tp.kp_angular), arr(tp.kd_angular)
    res = []
    for t in range(T):
        a1._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                            dv["ia"], dv["ig"]))
        a1._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                               rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
        a1._check(L.a1mpc_command_batch(eng.h, B, cs, dt, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], dv["ref"] if mpc else None, B, dv["des"], B))
        lvd = off(dv["ref"], 5 * B * 8) if mpc else off(dv["des"], 6 * B * 8)
        a1._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(tp.gait), dv["gc"], ds.speed, u["mode"], x0p(9), lvd, dv["rz"], dv["rot"], x0p(3),
                                            u["plan"], None, dv["trel"], None, None))
        a1._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, dt, dv["gc"], u["plan"], dv["rz"],
                                           dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        if t == 0:
            a1._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
        else:
            a1._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, dt, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                               ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        if mpc:
            a1._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
            if warm is not None:
                a1._check(L.a1mpc_solve_batch_warm(eng.h, B, C.byref(inp), C.byref(out), warm, 0))
            else:
                a1._check(L.a1mpc_solve_batch(eng.h, B, C.byref(inp), C.byref(out)))
        else:
            a1._check(L.a1mpc_stance_qp_batch(eng.h, B, C.c_size_t(B), dv["x0"], dv["rot"], dv["rz"], dv["foot"], u["contact"], dv["des"], dv["kpl"],
                                              kdl.ctypes.data, kpa.ctypes.data, kda.ctypes.data, dv["f_body"], u["status"], None))
        a1._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        src = dict(tau=dv["tau"], f_body=dv["f_body"], status=u["status"], contacts=u["contact"], movement_mode=u["mode"], x0=dv["x0"], ref=dv["ref"])
        res.append({k: d2h(a1, eng, src[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in OUT_SPECS if mpc or k != "ref"})
    for p in list(dv.values()) + list(u.values()) + [imu, sw, ekf, warm, cs]:
        if p is not None:
            L.a1mpc_device_free(eng.h, p)
    return res


def tick_run_device(a1, eng, tick, ds, B, T, dt, t0=0):
    """ticks t0 .. T-1 of `tick` on device pointers; one dict of host outputs per tick"""
    L = a1.lib()
    mpc = tick.params.mode == a1.TICK_MPC
    keys = [k for k in OUT_SPECS if mpc or k != "ref"]
    d = {k: eng.dalloc(int(np.prod(OUT_SPECS[k][0] + (B,))) * np.dtype(OUT_SPECS[k][1]).itemsize) for k in keys}
    outs = a1.TickOutputs(*[d.get(k) for k in a1.TICK_OUTPUTS])
    res = []
    for t in range(t0, T):
        ins = a1.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1.TICK_INPUTS])
        tick.run_ptrs(dt, ins, outs)
        res.append({k: d2h(a1, eng, d[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in keys})
    for p in d.values():
        L.a1mpc_device_free(eng.h, p)
    return res


def first_difference(got, want):
    """None when every output of every tick is bit-identical, else (tick, name, count of differing elements)"""
    assert len(got) == len(want)
    for t, (g, w) in enumerate(zip(got, want)):
        assert g.keys() == w.keys()
        for k in g:
            if g[k].tobytes() != w[k].tobytes():
                return t, k, int((g[k].view(np.uint8).reshape(-1, g[k].itemsize) != w[k].view(np.uint8).reshape(-1, w[k].itemsize)).any(axis=1).sum())
    return None
