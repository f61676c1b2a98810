"""dev tool: cost of a1mpc_tick_reset_robots on device masks, with the Gazebo MPC tick (held pattern, horizon 10) on device pointers.

  python tools/tick_reset_bench.py [--sizes 1024,16384,65536] [--repeats 7] [--calls 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) device time of one a1mpc_tick_reset_robots with 0 %, 1 %, 10 % and 100 % of the robots masked (random robots), and of one
      a1mpc_tick_reset: `calls` back-to-back calls between two CUDA events, the mean per call; the median, min and max over the repeats;
  (b) the run that follows a partial reset against a run with nothing pending: single runs between two CUDA events, recorded after the
      reset was enqueued, alternating the two on the same walking state; the median, min and max over `calls` x `repeats` runs of each.
      The reset is all-zero, so the two runs differ only by the launch of ekf_init_pending: a reset that does flag robots changes their
      state, and with it what the rest of the run costs, so a run after it cannot be matched against a run on the same state;
  (c) the device time of the two new kernels (tick_reset_robots_kernel, ekf_init_pending) per fraction from torch.profiler's CUDA activity
      trace of `calls` resets and runs (a run of its own: the profiler slows the host).  ekf_init_pending is what the run after a partial
      reset adds to a run with nothing pending;
  (d) host time to enqueue one a1mpc_tick_reset_robots on a device mask (perf_counter around the call, after a synchronise so that the
      stream's queue is empty); the median, min and max over `calls` x `repeats` calls.
Inputs: tests/tick_scenarios.py; the tick runs 8 ticks (walking from tick 5) before anything is timed, and every timed run takes tick 7's
inputs.  Not part of bench.py's contract."""
import argparse
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
from tick_scenarios import DeviceSeqs, h2d, tick_inputs

FRACTIONS = (0.0, 0.01, 0.1, 1.0)
WARM_TICKS = 8


def device_line():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    if q.returncode != 0:
        raise RuntimeError("nvidia-smi failed: %s" % q.stderr.strip())
    return q.stdout.strip()


def stats(v):
    v = np.array(v)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def window_ms(eng, fn, k):
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


def kernel_us(eng, fn, k, names):
    """device time per call (us) of the kernels whose name contains one of `names`, from torch.profiler's CUDA activity trace of k calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(k):
            fn()
        eng.sync()
    out = {n: 0.0 for n in names}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        for n in names:
            if n in e.key:
                out[n] += us / k
    return out


def bench_size(eng, B, repeats, calls):
    seqs, speed = tick_inputs(B, WARM_TICKS, 5)
    ds = DeviceSeqs(a1mpc, eng, seqs, speed)
    tick = a1mpc.Tick(eng, B, a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC))
    L = a1mpc.lib()
    keys = ("tau", "f_body", "status", "contacts", "movement_mode", "x0", "ref")
    size = dict(tau=96, f_body=96, status=4, contacts=4, movement_mode=4, x0=96, ref=72)
    outp = {k: eng.dalloc(size[k] * B) for k in keys}
    outs = a1mpc.TickOutputs(*[outp[k] for k in a1mpc.TICK_OUTPUTS])
    rng = np.random.default_rng(B)
    masks = {}
    for f in FRACTIONS:
        m = np.zeros(B, np.uint8)
        m[rng.choice(B, int(round(f * B)), replace=False)] = 1
        p = eng.dalloc(B)
        h2d(a1mpc, eng, p, m)
        masks[f] = p
    ins_at = lambda t: a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS])
    last = ins_at(WARM_TICKS - 1)
    run = lambda: tick.run_ptrs(DT, last, outs)
    try:
        for t in range(WARM_TICKS):
            tick.run_ptrs(DT, ins_at(t), outs)
        eng.sync()
        # (a) reset calls; a run after each round clears the pending flags and the full reset's EKF re-init
        reset_ms = {f: [] for f in FRACTIONS}
        reset_ms["full"] = []
        for _ in range(repeats):
            for f in FRACTIONS:
                reset_ms[f].append(window_ms(eng, lambda f=f: tick.reset_robots_ptr(masks[f].value), calls))
                run()
            reset_ms["full"].append(window_ms(eng, tick.reset, calls))
            run()
        eng.sync()
        # (b) the run after an all-zero partial reset against a run with nothing pending, alternating
        for _ in range(calls):
            run()
        run_ms = {"none": [], "pending": []}
        e0, e1 = eng.event(), eng.event()
        for _ in range(repeats):
            for _ in range(calls):
                for key in ("none", "pending"):
                    if key == "pending":
                        tick.reset_robots_ptr(masks[0.0].value)
                    eng.record(e0)
                    run()
                    eng.record(e1)
                    run_ms[key].append(eng.elapsed_ms(e0, e1))
        for e in (e0, e1):
            L.a1mpc_event_destroy(eng.h, e)
        # (d) host enqueue time of a reset on a device mask
        enq = []
        for _ in range(repeats * calls):
            eng.sync()
            t0 = time.perf_counter()
            tick.reset_robots_ptr(masks[0.1].value)
            enq.append((time.perf_counter() - t0) * 1e3)
        run()
        eng.sync()
        # (c) kernel times from the profiler
        kern = {}
        for f in FRACTIONS:
            def step(f=f):
                tick.reset_robots_ptr(masks[f].value)
                run()
            kern[f] = kernel_us(eng, step, calls, ("tick_reset_robots_kernel", "ekf_init_pending", "ekf_update_kernel"))
    finally:
        eng.sync()
        tick.close()
        ds.free()
        for p in list(outp.values()) + list(masks.values()):
            L.a1mpc_device_free(eng.h, p)
    return dict(B=B, reset_ms={str(k): stats(v) for k, v in reset_ms.items()}, run_ms={k: stats(v) for k, v in run_ms.items()},
                run_extra_ms_median=float(np.median(run_ms["pending"]) - np.median(run_ms["none"])),
                kernel_us_per_call={str(f): v for f, v in kern.items()},
                enqueue_ms=stats(enq))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,16384,65536")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the record here")
    a = ap.parse_args()
    dev = device_line()
    print("device:", dev, flush=True)
    eng = a1mpc.Engine(a1mpc.default_config(horizon=10))
    rec = dict(device=dev, repeats=a.repeats, calls=a.calls, results=[])
    try:
        for B in (int(s) for s in a.sizes.split(",")):
            r = bench_size(eng, B, a.repeats, a.calls)
            rec["results"].append(r)
            f = lambda d: "%.4f [%.4f, %.4f]" % (d["median"], d["min"], d["max"])
            print("B=%6d  reset_robots ms: " % B + ", ".join("%s%% %s" % (round(100 * x), f(r["reset_ms"][str(x)])) for x in FRACTIONS) +
                  " | full reset %s" % f(r["reset_ms"]["full"]), flush=True)
            print("          run ms: nothing pending %s, after an all-zero partial reset %s (difference of the medians %+.4f)" %
                  (f(r["run_ms"]["none"]), f(r["run_ms"]["pending"]), r["run_extra_ms_median"]), flush=True)
            print("          kernels us/call: " + "; ".join("%s%%: %s" % (round(100 * x), ", ".join("%s %.2f" % kv for kv in r["kernel_us_per_call"][str(x)].items()))
                                                       for x in FRACTIONS), flush=True)
            print("          enqueue ms %s" % f(r["enqueue_ms"]), flush=True)
    finally:
        eng.close()
    print(json.dumps(rec))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
