"""dev tool: device time of one MPC-mode control tick, a1mpc_tick_run against the same stages called one by one, on device pointers.

  python tools/tick_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--ticks 20] [--json PATH] [--sched]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) the staged chain: orientation -> leg kinematics -> command -> update_plan -> swing legs -> EKF update -> terrain pitch -> warm solve
      (a1mpc_solve_batch_warm, shift 0, no schedule) -> joint torques, ten entry points;
  (b) a1mpc_tick_run with the Gazebo MPC parameters (the same stages; orientation + command and kinematics + update_plan + swing fused);
  (a) and (b) alternate over the repeats, `ticks` ticks each between two CUDA events;
  (c) a per-stage breakdown of (a): one more window of `ticks` back-to-back ticks with an event at every stage boundary, no
      synchronisation inside; each stage's mean over the ticks (the means add up to the window's tick mean) and its per-tick range;
  (d) host time to enqueue one tick in (a) and in (b) (perf_counter around the calls, no synchronisation inside; the median over `ticks`
      ticks, each after a synchronise so that the stream's queue is empty);
  (e) the device time of the kernels, memsets and copies of (a) and of (b) per stage, per tick, from torch.profiler's CUDA activity trace
      of `ticks` ticks (a run of its own: the profiler slows the host).
(a) and (b) report the median, min and max over the repeats of each window's mean tick time.
With --sched the run times the scheduled tick instead (gait.horizon = the handle's horizon: the solve on update_plan's schedule with step 0
the swing stage's contacts, a1mpc_solve_batch_ext_warm with shift 1) against the held-pattern tick (gait.horizon = 0), two a1mpc.Tick
objects on the same inputs, alternating windows as in (a) / (b), and (e) for both.
Inputs: tests/tick_scenarios.py, with every robot walking from tick 5 to tick `ticks` - 5 of each window, so that every window of
`ticks` ticks does the same work.  Not part of bench.py's contract."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200")); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import a1mpc
from command_scenarios import DT
from tick_scenarios import DeviceSeqs, h2d, off, tick_inputs


def device_line():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    return q.stdout.strip()


def stats(ms):
    ms = np.array(ms)
    return dict(ms_min=float(ms.min()), ms_median=float(np.median(ms)), ms_max=float(ms.max()))


STAGES = ("orientation", "kinematics", "command", "update_plan", "swing", "ekf", "terrain", "solve", "torques")
# kernel name -> stage of (e); every other kernel and memset of a tick belongs to the solve (pack_kernel, the class kernels)
KERNEL_STAGE = (("tick_front_a", "front_a"), ("tick_front_b", "front_b"), ("tick_front_sched", "front_b"), ("orientation_kernel", "orientation"), ("leg_kinematics", "kinematics"),
                ("command_kernel", "command"), ("update_plan", "update_plan"), ("swing_legs", "swing"), ("ekf_", "ekf"), ("terrain_pitch", "terrain"),
                ("joint_torques", "torques"), ("Memcpy", "copies"))


def kernel_ms(eng, fn, k):
    """summed device time per stage of the kernels, memsets and copies of k calls of fn, per call (ms), from torch.profiler's CUDA activity
    trace.  The four solve class kernels run concurrently on their own streams, so the solve's sum can exceed its span."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(k):
            fn()
        eng.sync()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        stage = next((st for key, st in KERNEL_STAGE if key in e.key), "solve")
        out[stage] = out.get(stage, 0.0) + us / 1e3 / k
    out["all"] = sum(out.values())
    return out


def window_inputs(eng, B, T):
    """tests/tick_scenarios.py's inputs with one period per window: every robot starts walking at tick 5 and stops at tick T - 5"""
    seqs, speed = tick_inputs(B, T, B)
    seqs["cmd"][:, 6] = 0.0
    seqs["cmd"][5, 6] = 1.0
    seqs["cmd"][T - 5, 6] = 1.0
    return DeviceSeqs(a1mpc, eng, seqs, speed)


def timed(eng, fn, k):
    """mean device ms per call of k back-to-back calls of fn, between two CUDA events"""
    e0, e1 = eng.event(), eng.event()
    eng.record(e0)
    for _ in range(k):
        fn()
    eng.record(e1)
    ms = eng.elapsed_ms(e0, e1) / k
    for e in (e0, e1):
        a1mpc.lib().a1mpc_event_destroy(eng.h, e)
    return ms


def bench_sched(eng, B, repeats, ticks):
    """--sched: the held-pattern tick against the scheduled tick, same inputs, alternating windows of `ticks` ticks"""
    T = ticks
    ds = window_inputs(eng, B, T)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    dtau = eng.dalloc(12 * B * 8)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    runs = {}
    for name, horizon in (("held", 0), ("sched", eng.cfg.horizon)):
        tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
        tp.gait.horizon = horizon
        tick, n = a1mpc.Tick(eng, B, tp), [0]

        def run(tick=tick, n=n):
            t = n[0] % T
            n[0] += 1
            tick.run_ptrs(DT, tins[t], touts)
        runs[name] = (tick, run)
    for _ in range(T):   # warm-up: every shape of the timed window, the warm faces settled
        for _, run in runs.values():
            run()
    eng.sync()
    ms = {name: [] for name in runs}
    for _ in range(repeats):
        for name, (_, run) in runs.items():
            ms[name].append(timed(eng, run, T))
    kern = {name: kernel_ms(eng, run, T) for name, (_, run) in runs.items()}
    eng.sync()
    for tick, _ in runs.values():
        tick.close()
    a1mpc.lib().a1mpc_device_free(eng.h, dtau)
    ds.free()
    return dict(B=B, held=stats(ms["held"]), sched=stats(ms["sched"]), kernel_ms_per_tick=kern)


def bench_size(eng, B, repeats, ticks):
    L = a1mpc.lib()
    T = ticks
    tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
    # one period per window, so each window of T ticks starts from standstill and does the same work (the solve's cost depends strongly
    # on the stance mix: standstill is all four-stance)
    ds = window_inputs(eng, B, T)
    # (a): the staged chain's arrays and state
    nb = dict(rot=9, rz=9, x0=12, ia=3, ig=3, fpr=12, fvr=12, jac=36, foot=12, kpl=3, des=12, ref=9, gc=4, trel=12, fk=12, f_body=12, tau=12)
    dv = {k: eng.dalloc(n * B * 8) for k, n in nb.items()}
    for k in ("x0", "gc", "tau"):
        h2d(a1mpc, eng, dv[k], np.zeros((nb[k], B)))
    u = {k: eng.dalloc(B * 4) for k in ("mode", "plan", "contact", "status", "est", "est_status")}
    imu, sw, ekf, warm, cs = eng.imu_alloc(B), eng.swing_alloc(B), eng.dalloc(L.a1mpc_ekf_bytes(B)), eng.warm_alloc(B), eng.dalloc(L.a1mpc_command_bytes(B))
    a1mpc._check(L.a1mpc_command_init_batch(eng.h, B, cs, C.byref(tp.command), dv["ref"], B))
    x0p = lambda row: off(dv["x0"], row * B * 8)
    inp = a1mpc.Inputs(dv["x0"], dv["rot"], dv["foot"], dv["ref"], u["contact"], B)
    out = a1mpc.Outputs(dv["f_body"], u["status"], None, None, B)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    rho_opt, rho_fix, kp, kd, km, tg = (arr(getattr(tp, k)) for k in ("rho_opt", "rho_fix", "kp_foot", "kd_foot", "km_foot", "torques_gravity"))
    n = [0]

    def staged(mark=None):
        t = n[0] % T
        n[0] += 1
        mark = mark or (lambda i: None)
        a1mpc._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", t), ds.at("gyro", t), ds.at("acc", t), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                               dv["ia"], dv["ig"]))
        mark(1)
        a1mpc._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", t), ds.at("joint_vel", t), dv["rot"], rho_opt.ctypes.data,
                                                  rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
        mark(2)
        a1mpc._check(L.a1mpc_command_batch(eng.h, B, cs, DT, ds.at("cmd", t), x0p(3), B, u["mode"], dv["kpl"], dv["ref"], B, dv["des"], B))
        mark(3)
        a1mpc._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(tp.gait), dv["gc"], ds.speed, u["mode"], x0p(9), off(dv["ref"], 5 * B * 8), dv["rz"],
                                               dv["rot"], x0p(3), u["plan"], None, dv["trel"], None, None))
        mark(4)
        a1mpc._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(tp.gait), kp.ctypes.data, kd.ctypes.data, sw, DT, dv["gc"], u["plan"], dv["rz"],
                                              dv["foot"], dv["trel"], ds.at("foot_force", t), dv["fk"], u["contact"], None, None))
        mark(5)
        a1mpc._check(L.a1mpc_ekf_update_batch(eng.h, B, ekf, DT, tp.assume_flat_ground, u["mode"], dv["ia"], dv["ig"], dv["rot"], dv["fpr"], dv["fvr"],
                                              ds.at("foot_force", t), x0p(3), x0p(9), u["est"], u["est_status"]))
        mark(6)
        a1mpc._check(L.a1mpc_terrain_pitch_batch(eng.h, B, sw, tp.use_terrain_adapt, x0p(3), dv["ref"], B, None))
        mark(7)
        a1mpc._check(L.a1mpc_solve_batch_warm(eng.h, B, C.byref(inp), C.byref(out), warm, 0))
        mark(8)
        a1mpc._check(L.a1mpc_joint_torques_batch(eng.h, B, dv["f_body"], dv["fk"], dv["jac"], u["contact"], km.ctypes.data, tg.ctypes.data, dv["tau"]))
        mark(9)

    # (b): the tick
    tick = a1mpc.Tick(eng, B, tp)
    dtau = eng.dalloc(12 * B * 8)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    m = [0]

    def fused():
        t = m[0] % T
        m[0] += 1
        tick.run_ptrs(DT, tins[t], touts)

    # first tick of the chain: EKF init, as the tick's first run does
    a1mpc._check(L.a1mpc_orientation_batch(eng.h, B, ds.at("quat", 0), ds.at("gyro", 0), ds.at("acc", 0), imu, dv["rot"], dv["rz"], dv["x0"], B,
                                           dv["ia"], dv["ig"]))
    a1mpc._check(L.a1mpc_leg_kinematics_batch(eng.h, B, ds.at("joint_pos", 0), ds.at("joint_vel", 0), dv["rot"], rho_opt.ctypes.data,
                                              rho_fix.ctypes.data, dv["fpr"], dv["jac"], dv["fvr"], dv["foot"], None))
    a1mpc._check(L.a1mpc_ekf_init_batch(eng.h, B, ekf, dv["fpr"], dv["rot"]))
    for _ in range(T):   # warm-up: every shape of the timed window, the warm faces settled
        staged()
        fused()
    eng.sync()

    ta, tb = [], []
    for _ in range(repeats):
        ta.append(timed(eng, staged, T))
        tb.append(timed(eng, fused, T))
    # (c) per-stage breakdown of (a): one window of T back-to-back ticks, as (a) times them, with an event at every stage boundary and no
    # synchronisation inside; a stage's time is the interval from the previous boundary to its own, so the intervals add up to the window
    ev = [eng.event() for _ in range(len(STAGES) * T + 1)]
    k = [0]

    def mark(i):
        k[0] += 1
        eng.record(ev[k[0]])

    eng.record(ev[0])
    for _ in range(T):
        staged(mark)
    eng.sync()
    per = np.array([[eng.elapsed_ms(ev[t * len(STAGES) + i], ev[t * len(STAGES) + i + 1]) for i in range(len(STAGES))] for t in range(T)])
    for e in ev:
        L.a1mpc_event_destroy(eng.h, e)
    # (e) kernel time per stage, from the CUDA activity trace of T ticks of (a) and of (b), each in a profiler session of its own
    kern = dict(staged=kernel_ms(eng, staged, T), tick=kernel_ms(eng, fused, T))
    # (d) host enqueue time of one tick
    ha, hb = [], []
    for _ in range(T):
        eng.sync()
        t0 = time.perf_counter(); staged(); ha.append((time.perf_counter() - t0) * 1e3)
        eng.sync()
        t0 = time.perf_counter(); fused(); hb.append((time.perf_counter() - t0) * 1e3)
    eng.sync()
    tick.close()
    for p in list(dv.values()) + list(u.values()) + [imu, sw, ekf, warm, cs, dtau]:
        L.a1mpc_device_free(eng.h, p)
    ds.free()
    tick_ms = per.sum(axis=1)
    return dict(B=B, staged=stats(ta), tick=stats(tb),
                staged_stages_ms_mean={s: float(per[:, i].mean()) for i, s in enumerate(STAGES)},
                staged_stages_ms_per_tick_range={s: [float(per[:, i].min()), float(per[:, i].max())] for i, s in enumerate(STAGES)},
                instrumented_tick_ms=dict(mean=float(tick_ms.mean()), min=float(tick_ms.min()), max=float(tick_ms.max())),
                kernel_ms_per_tick=kern, enqueue_ms_median=dict(staged=float(np.median(ha)), tick=float(np.median(hb))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,16384,65536")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the record here")
    ap.add_argument("--sched", action="store_true", help="time the scheduled tick against the held-pattern tick")
    a = ap.parse_args()
    if a.ticks < 12:
        ap.error("--ticks must be at least 12 (standstill, walking, standstill in every window)")
    dev = device_line()
    print("device:", dev, flush=True)
    eng = a1mpc.Engine(a1mpc.default_config())
    rec = dict(device=dev, repeats=a.repeats, ticks=a.ticks, results=[], **(dict(mode="sched") if a.sched else {}))
    for B in [int(s) for s in a.sizes.split(",")]:
        if a.sched:
            r = bench_sched(eng, B, a.repeats, a.ticks)
            rec["results"].append(r)
            f = lambda k: "%.4f ms [%.4f-%.4f]" % (r[k]["ms_median"], r[k]["ms_min"], r[k]["ms_max"])
            print("B=%6d  held-pattern tick %s | scheduled tick %s" % (B, f("held"), f("sched")), flush=True)
            for w in ("held", "sched"):
                print("         (e) kernel time per tick, %s (ms): " % w + ", ".join("%s %.4f" % kv for kv in sorted(r["kernel_ms_per_tick"][w].items())),
                      flush=True)
            continue
        r = bench_size(eng, B, a.repeats, a.ticks)
        rec["results"].append(r)
        f = lambda k: "%.4f ms [%.4f-%.4f]" % (r[k]["ms_median"], r[k]["ms_min"], r[k]["ms_max"])
        print("B=%6d  staged chain %s | tick %s | enqueue staged %.3f ms, tick %.3f ms" % (B, f("staged"), f("tick"), r["enqueue_ms_median"]["staged"],
                                                                                           r["enqueue_ms_median"]["tick"]), flush=True)
        it = r["instrumented_tick_ms"]
        print("         (c) staged stages, mean per tick (ms): " + ", ".join("%s %.4f" % kv for kv in r["staged_stages_ms_mean"].items()) +
              " | instrumented tick mean %.4f [%.4f-%.4f]" % (it["mean"], it["min"], it["max"]), flush=True)
        print("         (c) per-tick range: " + ", ".join("%s %.4f-%.4f" % (s_, *v) for s_, v in r["staged_stages_ms_per_tick_range"].items()), flush=True)
        for w in ("staged", "tick"):
            print("         (e) kernel time per tick, %s (ms): " % w + ", ".join("%s %.4f" % kv for kv in sorted(r["kernel_ms_per_tick"][w].items())),
                  flush=True)
    print(json.dumps(rec))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
