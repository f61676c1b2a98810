"""dev tool: device time of the orientation and command stages (a1mpc_orientation_batch, a1mpc_command_batch) and of the whole control tick
from raw sensor arrays, on device pointers.

  python tools/command_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--iters 50] [--ticks 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) a1mpc_orientation_batch with the IMU filters, all outputs (rot, rot_z, x0 rows, imu_acc, imu_ang_vel);
  (b) a1mpc_command_batch with ref and des;
  (c) one MPC-mode tick of nine stages: orientation -> leg kinematics -> command -> update_plan -> swing legs -> EKF -> terrain pitch ->
      scheduled warm solve (a1mpc_solve_batch_ext_warm) -> joint torques.
(a) and (b) alternate over the repeats and are timed two ways: L2-warm, `iters` back-to-back calls between two CUDA events on the
handle's stream (the same state and arrays every call, so the working set stays in the 50 MB L2), and L2-cold, `iters` single calls each
after a1mpc_flush_l2 with its own event pair (the working set comes from HBM, as in a tick where other stages ran in between).  (c) is
`ticks` ticks per repeat.  Reports min / median / max ms per call and M robots/s.  Inputs: tests/command_scenarios.py.  Not part of
bench.py's contract."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200")); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import a1mpc
from command_scenarios import DT, command_sequence, imu_sequence


def device_line():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    return q.stdout.strip()


def upload(eng, x):
    x = np.ascontiguousarray(x)
    p = eng.dalloc(max(x.nbytes, 8))
    a1mpc._check(a1mpc.lib().a1mpc_memcpy_h2d(eng.h, p, x.ctypes.data, x.nbytes))
    return p


def timed(eng, fn, iters):
    e0, e1 = eng.event(), eng.event()
    eng.record(e0)
    for _ in range(iters):
        fn()
    eng.record(e1)
    ms = eng.elapsed_ms(e0, e1) / iters
    for e in (e0, e1):
        a1mpc.lib().a1mpc_event_destroy(eng.h, e)
    return ms


def timed_cold(eng, fn, iters):
    """median over `iters` single calls, each after a write of a buffer larger than L2, each between its own event pair"""
    e0, e1 = eng.event(), eng.event()
    ms = []
    for _ in range(iters):
        eng.flush_l2()
        eng.record(e0)
        fn()
        eng.record(e1)
        ms.append(eng.elapsed_ms(e0, e1))
    for e in (e0, e1):
        a1mpc.lib().a1mpc_event_destroy(eng.h, e)
    return float(np.median(ms))


def stats(ms, B):
    ms = np.array(ms)
    return dict(ms_min=float(ms.min()), ms_median=float(np.median(ms)), ms_max=float(ms.max()),
                mrobots_per_s_median=float(B / np.median(ms) / 1e3), mrobots_per_s_range=[float(B / ms.max() / 1e3), float(B / ms.min() / 1e3)])


def off(p, nbytes):
    return C.c_void_p(p.value + nbytes)


def bench_size(eng, B, repeats, iters, ticks, ptrs):
    L = a1mpc.lib()
    T = ticks
    rng = np.random.default_rng(B)
    quat, gyro, acc = imu_sequence(B, T, B, gimbal_share=0.0, gentle=True)
    cmd, _ = command_sequence(B, T, B + 1)
    q = np.tile(np.array([0.0, 0.8, -1.6] * 4)[None, :, None], (T, 1, B)) + 0.05 * rng.standard_normal((T, 12, B))
    dq = 0.5 * rng.standard_normal((T, 12, B))
    force = rng.uniform(0.0, 80.0, (T, 4, B))
    seqs = dict(quat=quat, gyro=gyro, acc=acc, cmd=cmd, q=q, dq=dq, force=force)
    ds = {k: upload(eng, v) for k, v in seqs.items()}
    at = lambda k, t: off(ds[k], t * seqs[k][0].nbytes)
    d = a1mpc.DeviceBatch(eng, B)
    a1mpc._check(L.a1mpc_memcpy_h2d(eng.h, d.x0, np.zeros((12, B)).ctypes.data, 12 * B * 8))
    nb = dict(rz=9, ia=3, ig=3, fpr=12, fvr=12, jac=36, kpl=3, des=12, gc=4, trel=12, fk=12, tau=12)
    dv = {k: upload(eng, np.zeros((n, B))) for k, n in nb.items()}
    d_sp = upload(eng, np.repeat(rng.choice([2.0, 3.0, 4.0], B)[None, :], 4, axis=0))
    d_mode, d_plan, d_sched, d_est, d_st = (eng.dalloc(n * B * 4) for n in (1, 1, 10, 1, 1))
    imu, sw, ekf, warm = eng.imu_alloc(B), eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B)), eng.warm_alloc(B)
    cs = eng.dalloc(L.a1mpc_command_bytes(B))
    cp = a1mpc.default_command_params()
    a1mpc._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(cp), d.ref, B))
    ptrs += list(ds.values()) + list(dv.values()) + [d_sp, d_mode, d_plan, d_sched, d_est, d_st, imu, sw, ekf, warm, cs]
    rho_fix = np.array([[0.1805, 0.047, 0.0838, 0.21, 0.21], [0.1805, -0.047, -0.0838, 0.21, 0.21],
                        [-0.1805, 0.047, 0.0838, 0.21, 0.21], [-0.1805, -0.047, -0.0838, 0.21, 0.21]]).reshape(20)
    rho_opt = np.zeros(12)
    gp = a1mpc.default_gait_params(10)
    kp, kd = np.array([300.0, 400, 400] * 4), np.array([8.0, 8, 8] * 4)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    ext = a1mpc.InputsExt(d_sched.value, None)
    x0p = lambda row: off(d.x0, row * B * 8)
    n = [0]

    def orientation():
        t = n[0] % T
        a1mpc._check(L.a1mpc_orientation_batch(eng.h, B, at("quat", t), at("gyro", t), at("acc", t), imu, d.rot, dv["rz"], d.x0, B, dv["ia"], dv["ig"]))

    def command():
        t = n[0] % T
        a1mpc._check(L.a1mpc_command_batch(eng.h, B, cs, DT, at("cmd", t), x0p(3), B, d_mode, dv["kpl"], d.ref, B, dv["des"], B))

    def tick():
        t = n[0] % T
        n[0] += 1
        orientation()
        a1mpc._check(L.a1mpc_leg_kinematics_batch(eng.h, B, at("q", t), at("dq", t), d.rot, rho_opt.ctypes.data, rho_fix.ctypes.data, dv["fpr"],
                                                  dv["jac"], dv["fvr"], d.foot, None))
        command()
        a1mpc._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(gp), dv["gc"], d_sp, d_mode, x0p(9), off(d.ref, 5 * B * 8), dv["rz"], d.rot, x0p(3),
                                               d_plan, d_sched, dv["trel"], None, None))
        a1mpc._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, DT, dv["gc"], d_plan, dv["rz"], d.foot,
                                              dv["trel"], at("force", t), dv["fk"], d.contact, None, None))
        a1mpc._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, DT, 1, d_mode, dv["ia"], dv["ig"], d.rot, dv["fpr"], dv["fvr"], at("force", t), x0p(3),
                                              x0p(9), d_est, d_st))
        a1mpc._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, 1, x0p(3), d.ref, B, None))
        a1mpc._check(L.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out), warm, 1))
        a1mpc._check(L.a1mpc_joint_torques_batch(eng.h, B, d.f_body, dv["fk"], dv["jac"], d.contact, km.ctypes.data, tg.ctypes.data, dv["tau"]))

    orientation()
    a1mpc._check(L.a1mpc_leg_kinematics_batch(eng.h, B, at("q", 0), at("dq", 0), d.rot, rho_opt.ctypes.data, rho_fix.ctypes.data, dv["fpr"], dv["jac"],
                                              dv["fvr"], d.foot, None))
    a1mpc._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], d.rot))
    for _ in range(T):
        tick()
    eng.sync()
    f, status = d.download()
    optimal = float((status == a1mpc.STATUS_OPTIMAL).mean())
    ta, tb, ca, cb = [], [], [], []
    for _ in range(repeats):
        ta.append(timed(eng, orientation, iters))
        tb.append(timed(eng, command, iters))
        ca.append(timed_cold(eng, orientation, iters))
        cb.append(timed_cold(eng, command, iters))
    tc = [timed(eng, tick, T) for _ in range(repeats)]
    d.free()
    return dict(B=B, last_tick_optimal_share=optimal, orientation=stats(ta, B), command=stats(tb, B), orientation_l2_cold=stats(ca, B),
                command_l2_cold=stats(cb, B), tick9=stats(tc, B))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,16384,65536")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the record here")
    a = ap.parse_args()
    dev = device_line()
    print("device:", dev, flush=True)
    eng = a1mpc.Engine(a1mpc.default_config())
    rec = dict(device=dev, repeats=a.repeats, iters=a.iters, ticks=a.ticks, results=[])
    ptrs = []
    for B in [int(s) for s in a.sizes.split(",")]:
        r = bench_size(eng, B, a.repeats, a.iters, a.ticks, ptrs)
        rec["results"].append(r)
        f = lambda k: "%.4f ms [%.4f-%.4f]" % (r[k]["ms_median"], r[k]["ms_min"], r[k]["ms_max"])
        print("B=%6d  L2-warm: orientation %s, command %s | L2-cold: orientation %s, command %s | 9-stage tick %.3f ms [%.3f-%.3f] | "
              "OPTIMAL %.2f %%" % (B, f("orientation"), f("command"), f("orientation_l2_cold"), f("command_l2_cold"), r["tick9"]["ms_median"],
                                   r["tick9"]["ms_min"], r["tick9"]["ms_max"], 100 * r["last_tick_optimal_share"]), flush=True)
        for p in ptrs:
            a1mpc.lib().a1mpc_device_free(eng.h, p)
        ptrs.clear()
    print(json.dumps(rec))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
