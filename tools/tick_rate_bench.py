"""dev tool: device time of the MPC-mode control tick whose solve runs on every period-th run of each robot (a1mpc_tick_set_mpc_period),
against the tick that never set a period, for the held pattern and the scheduled tick, on device pointers.

  python tools/tick_rate_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--ticks 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) one a1mpc.Tick per configuration (held / scheduled x period never set, 1, 2, 4, 10 with PLAYBACK_PLAN, and 4 with PLAYBACK_HOLD) on
      the same inputs; after a warm-up of `ticks` runs (longer than the first full period of every configuration) alternating windows of
      `ticks` back-to-back runs between two CUDA events; the median, min and max over the repeats of each window's mean time per run;
  (b) the device time per run of the solve (the pack kernels, class kernels and memsets) and of tick_rate_kernel, from torch.profiler's
      CUDA activity trace of `ticks` runs (a run of its own: the profiler slows the host);
  (c) the robots due per run in the timed windows, from the rule n % period == b % period.
Then, at B = 1024 over 40 runs, the staged chain of tests/test_gpu_tick_rate.py gives the share of due QPs that the warm guess certifies
(iters % 100 == 0: no interior-point iteration) and how many due QPs had a last solve fewer than `period` runs before (a robot's first
cycle), for periods 1 and 4.  Inputs: the stand / walk / stand window of tools/tick_bench.py.  Not part of bench.py's contract."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tick_bench as TB  # noqa: E402  (puts the package and tests/ on sys.path)
import a1mpc  # noqa: E402
from command_scenarios import DT  # noqa: E402

TB.KERNEL_STAGE = TB.KERNEL_STAGE + (("tick_rate_kernel", "rate"),)
CONFIGS = (("never", None, a1mpc.PLAYBACK_PLAN), ("p1", 1, a1mpc.PLAYBACK_PLAN), ("p2", 2, a1mpc.PLAYBACK_PLAN), ("p4", 4, a1mpc.PLAYBACK_PLAN),
           ("p10", 10, a1mpc.PLAYBACK_PLAN), ("p4_hold", 4, a1mpc.PLAYBACK_HOLD))


def due_per_run(B, period, first, count):
    """mean robots due per run over runs first .. first + count - 1 since the last set_mpc_period"""
    if not period or period == 1:
        return float(B)
    b = np.arange(B)
    return float(np.mean([((n == 0) | (n % period == b % period)).sum() for n in range(first, first + count)]))


def bench_size(eng, B, repeats, ticks):
    T = ticks
    ds = TB.window_inputs(eng, B, T)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    dtau = eng.dalloc(12 * B * 8)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    runs = {}
    for kind in ("held", "sched"):
        for name, period, playback in CONFIGS:
            tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
            tp.gait.horizon = eng.cfg.horizon if kind == "sched" else 0
            tick, n = a1mpc.Tick(eng, B, tp), [0]
            if period is not None:
                tick.set_mpc_period(period, playback)

            def run(tick=tick, n=n):
                t = n[0] % T
                n[0] += 1
                tick.run_ptrs(DT, tins[t], touts)
            runs["%s_%s" % (kind, name)] = (tick, run, period)
    for _ in range(T):   # warm-up: every shape of the timed window, the warm faces settled, the first full period over
        for _, run, _ in runs.values():
            run()
    eng.sync()
    ms = {name: [] for name in runs}
    for _ in range(repeats):
        for name, (_, run, _) in runs.items():
            ms[name].append(TB.timed(eng, run, T))
    kern = {name: TB.kernel_ms(eng, run, T) for name, (_, run, _) in runs.items()}
    due = {name: due_per_run(B, period, T, T) for name, (_, _, period) in runs.items()}
    eng.sync()
    for tick, _, _ in runs.values():
        tick.close()
    a1mpc.lib().a1mpc_device_free(eng.h, dtau)
    ds.free()
    return dict(B=B, ms={k: TB.stats(v) for k, v in ms.items()}, kernel_ms_per_tick=kern, due_per_run=due)


def warm_census(eng, B=1024, T=40):
    """the staged chain's due QPs: share certified by the warm guess, and the QPs whose last solve was fewer than `period` runs before"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_tick_rate import staged_chain_rate
    from tick_scenarios import DeviceSeqs, tick_inputs
    out = {}
    seqs, speed = tick_inputs(B, T, 5)
    ds = DeviceSeqs(a1mpc, eng, seqs, speed)
    try:
        for kind in ("held", "sched"):
            tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
            tp.gait.horizon = eng.cfg.horizon if kind == "sched" else 0
            for period in (1, 4):
                chain = staged_chain_rate(a1mpc, eng, tp, ds, B, T, DT, [period] * T, a1mpc.PLAYBACK_PLAN, record=True)
                last = np.zeros(B, np.int64)   # run 0 solves every robot
                hits = qps = early = early_hits = 0
                for t in range(1, T):
                    d, it = chain[t]["due"], chain[t]["iters"]
                    ok = (it % 100) == 0
                    hits += int(ok.sum()); qps += int(d.sum())
                    e = (t - last)[d] < period
                    early += int(e.sum()); early_hits += int(ok[e].sum())
                    last = np.where(d, t, last)
                out["%s_p%d" % (kind, period)] = dict(due_qps=qps, warm_certified=hits / qps, first_cycle_qps=early,
                                                      first_cycle_certified=(early_hits / early) if early else None)
    finally:
        ds.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,16384,65536")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    rec = dict(device=TB.device_line(), ticks=a.ticks, repeats=a.repeats, results=[])
    print("device: %s" % rec["device"], flush=True)
    eng = a1mpc.Engine(a1mpc.default_config())
    for B in [int(s) for s in a.sizes.split(",")]:
        r = bench_size(eng, B, a.repeats, a.ticks)
        rec["results"].append(r)
        for k in r["ms"]:
            m, kk = r["ms"][k], r["kernel_ms_per_tick"][k]
            print("B=%6d %-14s %.4f ms [%.4f-%.4f]  solve kernels %.4f ms  rate kernel %.4f ms  due/run %.0f" % (
                B, k, m["ms_median"], m["ms_min"], m["ms_max"], kk.get("solve", 0.0), kk.get("rate", 0.0), r["due_per_run"][k]), flush=True)
    rec["warm_census"] = warm_census(eng)
    for k, v in rec["warm_census"].items():
        print("warm census %s: %s" % (k, v), flush=True)
    eng.close()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
