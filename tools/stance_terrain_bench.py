"""dev tool: device time of the QP-mode stance QP on terrain normals against world-z pyramids, on device pointers.

  python tools/stance_terrain_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--iters 20] [--ticks 40] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) a1mpc_stance_qp_batch against a1mpc_stance_qp_batch_ext with all-e_z normals and with tilted per-foot normals (up to 0.6 rad, the
      generator of tests/test_emu_stance_terrain.py), on tools/stance_bench.py's robots (gazebo QP gains, the 16 contact masks uniform);
      each repeat is `iters` calls between two CUDA events, the three alternating;
  (b) the Gazebo QP-mode tick with FLAT against ESTIMATED (a1mpc_tick_set_stance_terrain) on tools/tick_bench.py's window: standstill,
      walking from tick 5, standstill for the last 5 ticks; each repeat is one window, the two ticks alternating;
  and the device time of surface_normals_kernel per tick from torch.profiler's CUDA activity trace, in a run of its own.
Reports min / median / max ms per call and the status counts.  Not part of bench.py's contract."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200")); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import a1mpc  # noqa: E402
from command_scenarios import DT  # noqa: E402
from stance_scenarios import gains, robots  # noqa: E402
from test_emu_stance_terrain import ez_normals, tilted_normals  # noqa: E402
from tick_scenarios import DeviceSeqs, tick_inputs  # noqa: E402

FIELDS = ("x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear")


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


def stats(ms):
    ms = np.array(ms)
    return dict(ms_min=float(ms.min()), ms_median=float(np.median(ms)), ms_max=float(ms.max()))


def bench_qp(eng, B, repeats, iters, free):
    L = a1mpc.lib()
    _, kdl, kpa, kda = gains("gazebo")
    st = robots(B, 2026 + B, "gazebo")
    d = {k: upload(eng, st[k]) for k in FIELDS}
    d_ez, d_tilt = upload(eng, ez_normals(B)), upload(eng, tilted_normals(B, 7 + B))
    d_f, d_s = eng.dalloc(12 * B * 8), eng.dalloc(B * 4)
    free += list(d.values()) + [d_ez, d_tilt, d_f, d_s]
    g = [v.ctypes.data for v in (kdl, kpa, kda)]
    qp = lambda: (eng.h, B, C.c_size_t(B), d["x0"], d["rot"], d["rot_z"], d["foot"], d["contact"], d["des"], d["kp_linear"], *g)
    calls = dict(world_z=lambda: a1mpc._check(L.a1mpc_stance_qp_batch(*qp(), d_f, d_s, None)),
                 ext_ez=lambda: a1mpc._check(L.a1mpc_stance_qp_batch_ext(*qp(), d_ez, d_f, d_s, None)),
                 ext_tilted=lambda: a1mpc._check(L.a1mpc_stance_qp_batch_ext(*qp(), d_tilt, d_f, d_s, None)))
    counts = {}
    for name, fn in calls.items():   # warm-up, and the status counts of each
        fn()
        status = np.zeros(B, dtype=np.int32)
        a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, status.ctypes.data, d_s, status.nbytes))
        eng.sync()
        counts[name] = np.bincount(status, minlength=5).tolist()
    ms = {name: [] for name in calls}
    for _ in range(repeats):
        for name, fn in calls.items():
            ms[name].append(timed(eng, fn, iters))
    return {name: dict(stats(v), statuses=counts[name]) for name, v in ms.items()}


def bench_tick(eng, B, repeats, T, free):
    seqs, speed = tick_inputs(B, T, B)
    seqs["cmd"][:, 6] = 0.0
    seqs["cmd"][5, 6] = 1.0
    seqs["cmd"][T - 5, 6] = 1.0
    ds = DeviceSeqs(a1mpc, eng, seqs, speed)
    tins = [a1mpc.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1mpc.TICK_INPUTS]) for t in range(T)]
    dtau = eng.dalloc(12 * B * 8)
    free.append(dtau)
    touts = a1mpc.TickOutputs(dtau, None, None, None, None, None, None)
    runs = {}
    for name, src in (("flat", a1mpc.TERRAIN_FLAT), ("estimated", a1mpc.TERRAIN_ESTIMATED)):
        tick, n = a1mpc.Tick(eng, B, a1mpc.default_tick_params(a1mpc.VARIANT_GAZEBO, a1mpc.TICK_QP)), [0]
        tick.set_stance_terrain(src)

        def run(tick=tick, n=n):
            tick.run_ptrs(DT, tins[n[0] % T], touts)
            n[0] += 1
        runs[name] = (tick, run)
    for _ in range(T):
        for _, run in runs.values():
            run()
    eng.sync()
    ms = {name: [] for name in runs}
    for _ in range(repeats):
        for name, (_, run) in runs.items():
            ms[name].append(timed(eng, run, T))
    kern = surface_normals_ms(eng, runs["estimated"][1], T)
    for tick, _ in runs.values():
        tick.close()
    ds.free()
    return dict({name: stats(v) for name, v in ms.items()}, surface_normals_kernel_ms_per_tick=kern)


def surface_normals_ms(eng, fn, k):
    """device ms per call of surface_normals_kernel over k calls of fn, from torch.profiler's CUDA activity trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(k):
            fn()
        eng.sync()
    for e in prof.key_averages():
        if "surface_normals_kernel" in e.key:
            us = getattr(e, "device_time_total", None)
            return (us if us is not None else e.cuda_time_total) / 1e3 / k
    raise RuntimeError("surface_normals_kernel not found in the trace")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,16384,65536")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--json")
    a = ap.parse_args()
    dev = device_line()
    eng = a1mpc.Engine(a1mpc.default_config(mass=gains("gazebo")[0]))
    res = dict(device=dev, sizes=[])
    free = []
    try:
        for B in [int(s) for s in a.sizes.split(",")]:
            r = dict(B=B, stance_qp=bench_qp(eng, B, a.repeats, a.iters, free), tick=bench_tick(eng, B, a.repeats, a.ticks, free))
            res["sizes"].append(r)
            q, t = r["stance_qp"], r["tick"]
            print("B=%6d  stance QP ms median [min-max]: world z %.3f [%.3f-%.3f], e_z %.3f [%.3f-%.3f], tilted %.3f [%.3f-%.3f]; statuses %s"
                  % (B, *[q[n][s] for n in ("world_z", "ext_ez", "ext_tilted") for s in ("ms_median", "ms_min", "ms_max")],
                     {n: q[n]["statuses"] for n in q}))
            print("          QP tick ms median [min-max]: FLAT %.3f [%.3f-%.3f], ESTIMATED %.3f [%.3f-%.3f]; surface_normals_kernel %.4f ms/tick"
                  % (*[t[n][s] for n in ("flat", "estimated") for s in ("ms_median", "ms_min", "ms_max")], t["surface_normals_kernel_ms_per_tick"]))
    finally:
        for p in free:
            a1mpc.lib().a1mpc_device_free(eng.h, p)
        eng.close()
    print("device: %s" % dev)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
