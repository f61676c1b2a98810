"""dev tool: device time of the MPC-mode control tick with world-z friction pyramids (A1MPC_TERRAIN_FLAT, the default) against the tick whose
pyramids stand on the estimated walking surface (A1MPC_TERRAIN_ESTIMATED), for the held pattern (gait.horizon = 0) and the scheduled tick
(gait.horizon = the handle's horizon), on device pointers.

  python tools/terrain_tick_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--ticks 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) four a1mpc.Tick objects with the Gazebo MPC parameters on the same inputs (held / scheduled x FLAT / ESTIMATED), alternating windows of
      `ticks` back-to-back ticks between two CUDA events; the median, min and max over the repeats of each window's mean tick time;
  (b) the device time of the kernels, memsets and copies of each tick per stage, per tick, from torch.profiler's CUDA activity trace of
      `ticks` ticks (a run of its own: the profiler slows the host); "terrain" is terrain_pitch_kernel or terrain_normals_kernel.
Inputs: the stand / walk / stand window of tools/tick_bench.py (every robot walks from tick 5 to tick `ticks` - 5 of each window, so every
window does the same work).  Not part of bench.py's contract."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tick_bench as TB  # noqa: E402  (puts the package and tests/ on sys.path)
import a1mpc  # noqa: E402
from command_scenarios import DT  # noqa: E402

TB.KERNEL_STAGE = TB.KERNEL_STAGE + (("terrain_normals", "terrain"),)
KINDS = (("held_flat", 0, a1mpc.TERRAIN_FLAT), ("held_estimated", 0, a1mpc.TERRAIN_ESTIMATED), ("sched_flat", None, a1mpc.TERRAIN_FLAT),
         ("sched_estimated", None, a1mpc.TERRAIN_ESTIMATED))


def bench_size(eng, B, repeats, ticks):
    T = ticks
    ds = TB.window_inputs(eng, B, T)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    dtau = eng.dalloc(12 * B * 8)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    runs = {}
    for name, horizon, source in KINDS:
        tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
        tp.gait.horizon = eng.cfg.horizon if horizon is None else horizon
        tick, n = a1mpc.Tick(eng, B, tp), [0]
        tick.set_terrain(source)

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
            ms[name].append(TB.timed(eng, run, T))
    kern = {name: TB.kernel_ms(eng, run, T) for name, (_, run) in runs.items()}
    eng.sync()
    for tick, _ in runs.values():
        tick.close()
    a1mpc.lib().a1mpc_device_free(eng.h, dtau)
    ds.free()
    return dict(B=B, ms={k: TB.stats(v) for k, v in ms.items()}, kernel_ms_per_tick=kern)


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
        f = lambda k: "%.4f ms [%.4f-%.4f]" % (r["ms"][k]["ms_median"], r["ms"][k]["ms_min"], r["ms"][k]["ms_max"])
        print("B=%6d  " % B + " | ".join("%s %s" % (k, f(k)) for k, _, _ in KINDS), flush=True)
        for k, _, _ in KINDS:
            print("         (b) kernel time per tick, %s (ms): " % k + ", ".join("%s %.4f" % kv for kv in sorted(r["kernel_ms_per_tick"][k].items())),
                  flush=True)
    print(json.dumps(rec))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
