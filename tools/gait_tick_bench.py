"""dev tool: device time of the MPC-mode control tick with per-robot gaits (a1mpc_tick_set_gaits), per gait, against the tick that never set
gaits, for the held pattern and the scheduled tick, on device pointers.

  python tools/gait_tick_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--ticks 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run: one a1mpc.Tick per
configuration (held / scheduled x gaits never set; every robot on the unshifted trot row ("trot1": the contact mix of "never" on the gait
path, so the two columns differ by the gait path alone); and every robot on the trot, pace, bound, pronk or walk row of a1mpc_gait_row, the
standstill offsets moved by 60 (b // 5 % 4) counts so that the batch holds every phase of the gait) on the same inputs; after a warm-up of
`ticks` runs, alternating windows of `ticks` back-to-back runs between two CUDA events; the median, min and max over the repeats of each
window's mean time per run; and the device time per run of the front kernel (tick_front_b / _sched or its gait twin) and of the solve from
torch.profiler's CUDA activity trace (a run of its own).  Inputs: the stand / walk / stand window of tools/tick_bench.py.  Not part of
bench.py's contract."""
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

GAITS = (("never", None), ("trot1", -a1mpc.GAIT_TROT), ("trot", a1mpc.GAIT_TROT), ("pace", a1mpc.GAIT_PACE), ("bound", a1mpc.GAIT_BOUND), ("pronk", a1mpc.GAIT_PRONK),
         ("walk", a1mpc.GAIT_WALK))


def rows_of(gtype, B):
    """gtype > 0: the row of a1mpc_gait_row in four phases; -GAIT_TROT: the trot row unshifted, the contact mix of "never" on the gait path"""
    rows = np.repeat(a1mpc.gait_row(abs(gtype))[:, None], B, axis=1)
    if gtype < 0:
        return np.ascontiguousarray(rows)
    rows[:4] = np.fmod(rows[:4] + 60.0 * ((np.arange(B) // 5) % 4)[None, :], rows[4][None, :])
    return np.ascontiguousarray(rows)


def bench_size(eng, B, repeats, ticks):
    T = ticks
    ds = TB.window_inputs(eng, B, T)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    dtau = eng.dalloc(12 * B * 8)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    runs = {}
    for kind in ("held", "sched"):
        for name, g in GAITS:
            tp = a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_MPC)
            tp.gait.horizon = eng.cfg.horizon if kind == "sched" else 0
            tick, n = a1mpc.Tick(eng, B, tp), [0]
            if g is not None:
                tick.set_gaits(rows_of(g, B))

            def run(tick=tick, n=n):
                t = n[0] % T
                n[0] += 1
                tick.run_ptrs(DT, tins[t], touts)
            runs["%s_%s" % (kind, name)] = (tick, run)
    for _ in range(T):
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
        for k in r["ms"]:
            m, kk = r["ms"][k], r["kernel_ms_per_tick"][k]
            print("B=%6d %-12s %.4f ms [%.4f-%.4f]  %s" % (B, k, m["ms_median"], m["ms_min"], m["ms_max"],
                                                          " ".join("%s %.4f" % (s, v) for s, v in sorted(kk.items()))), flush=True)
    eng.close()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
