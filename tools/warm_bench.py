"""dev tool: closed-loop throughput of the device-resident warm start next to the cold path.

  python tools/warm_bench.py [B] [noise]        a1mpc_solve_batch_warm against a1mpc_solve_batch (constant contact pattern)
  python tools/warm_bench.py [B] [noise] ext    a1mpc_solve_batch_ext_warm (shift 1) against a1mpc_solve_batch_ext

Constant pattern: a ring of T consecutive control ticks (state advanced by dt plus a random walk of sensor-level noise) is
uploaded once; the timed loop walks the ring.  Schedules (ext): T consecutive ticks of one gait -- the windows [t : t + 10] of a
horizon-20 schedule, terrain normals on -- with the state moved along the solver's own plan for one step (the first step of the
cold solution, through the oracle's condensed model) plus sensor-level noise; each lap starts from a reset buffer and the timed
part is ticks 1 .. T-1.  Not part of bench.py's contract (that measures independent QPs, i.e. the cold path)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200")); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import a1mpc

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
noise = float(sys.argv[2]) if len(sys.argv) > 2 else 0.1
EXT = len(sys.argv) > 3 and sys.argv[3] == "ext"
eng = a1mpc.Engine(a1mpc.default_config(horizon=10))
rng = np.random.default_rng(0)
scale = np.array([.02, .02, .02, .01, .01, .005, .1, .1, .1, .05, .05, .05])[:, None]
lib = a1mpc.lib()


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


print("device:", device_line(), flush=True)

if not EXT:
    T = 32
    st = a1mpc.gen_states(B, 2, 3)
    ticks = []
    for t in range(T):
        d = a1mpc.DeviceBatch(eng, B); d.upload(st); ticks.append(d)
        st = {k: v.copy() for k, v in st.items()}
        st["x0"][3:6] += 0.0025 * st["x0"][9:12]; st["x0"][0:3] += 0.0025 * st["x0"][6:9]
        st["x0"] += noise * rng.standard_normal(st["x0"].shape) * scale
    warm = eng.warm_alloc(B)

    def run(use_warm, reps):
        e0, e1 = eng.event(), eng.event()
        for t in range(T):   # warm-up lap
            if use_warm: a1mpc._check(lib.a1mpc_solve_batch_warm(eng.h, B, C.byref(ticks[t].inp), C.byref(ticks[t].out), warm, 0))
            else: eng.solve_ptrs(B, ticks[t].inp, ticks[t].out)
        eng.sync(); eng.record(e0)
        for r in range(reps):
            t = r % T
            if use_warm: a1mpc._check(lib.a1mpc_solve_batch_warm(eng.h, B, C.byref(ticks[t].inp), C.byref(ticks[t].out), warm, 0))
            else: eng.solve_ptrs(B, ticks[t].inp, ticks[t].out)
        eng.record(e1); eng.sync()
        return eng.elapsed_ms(e0, e1) / reps

    for name, w in (("cold", False), ("warm", True)):
        ms = run(w, 4 * T)
        f, status = ticks[(4 * T - 1) % T].download()
        print("B=%d noise %.2f %s: %.3f ms/tick  %.0f QPs/s  optimal %.4f" % (B, noise, name, ms, B / ms * 1e3, (status == 0).mean()), flush=True)
    sys.exit(0)

from common import obatch  # noqa: E402
from oracle import oracle_py as O  # noqa: E402

T, LAPS = 8, 4
st = a1mpc.gen_states(B, 4, 3)
s20, normals = a1mpc.gen_schedule(B, 20, 4, 3)
ocfg = O.make_config(horizon=10)
ticks = []
for t in range(T):
    sched = np.ascontiguousarray(s20[t:t + 10])
    st["contact"] = sched[0].copy()
    d = a1mpc.DeviceBatch(eng, B); d.upload(st)
    d_sched = eng.dalloc(sched.nbytes); a1mpc._check(lib.a1mpc_memcpy_h2d(eng.h, d_sched, sched.ctypes.data, sched.nbytes))
    d_norm = eng.dalloc(normals.nbytes); a1mpc._check(lib.a1mpc_memcpy_h2d(eng.h, d_norm, normals.ctypes.data, normals.nbytes))
    eng.sync()
    ticks.append((d, a1mpc.InputsExt(d_sched.value, d_norm.value)))
    f, status, iters, u = eng.solve_ext(st, sched, normals, want_u=True)
    ob = obatch(O, st)
    st = {k: v.copy() for k, v in st.items()}
    for b in range(B):
        r = O.rollout(ocfg, ob, b)
        st["x0"][:, b] = (r["A_d"] @ r["mpc_states"] + r["B_d_list"][:13] @ u[:12, b])[:12]
    st["x0"] += noise * rng.standard_normal(st["x0"].shape) * scale
warm = eng.warm_alloc(B)


def call(t, use_warm):
    d, ext = ticks[t]
    if use_warm: a1mpc._check(lib.a1mpc_solve_batch_ext_warm(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out), warm, 1))
    else: a1mpc._check(lib.a1mpc_solve_batch_ext(eng.h, B, C.byref(d.inp), C.byref(ext), C.byref(d.out)))


def run(use_warm):
    e0, e1 = eng.event(), eng.event()
    ms, hits, facts, opt = 0.0, [], [], []
    for lap in range(LAPS + 1):   # lap 0: warm-up
        a1mpc._check(lib.a1mpc_warm_reset(eng.h, warm, B))
        call(0, use_warm)
        eng.record(e0)
        for t in range(1, T):
            call(t, use_warm)
        eng.record(e1); eng.sync()
        if lap > 0:
            ms += eng.elapsed_ms(e0, e1)
    a1mpc._check(lib.a1mpc_warm_reset(eng.h, warm, B))
    call(0, use_warm)
    for t in range(1, T):   # counts of one more lap, tick by tick
        call(t, use_warm)
        d = ticks[t][0]
        f, status = d.download()
        it = np.zeros(B, dtype=np.int32)
        a1mpc._check(lib.a1mpc_memcpy_d2h(eng.h, it.ctypes.data, d.iters, it.nbytes)); eng.sync()
        hits.append(((it % 100) == 0).mean()); facts.append((it % 100 + it // 100).mean()); opt.append((status == 0).mean())
    return ms / (LAPS * (T - 1)), np.mean(hits), np.mean(facts), min(opt)


for name, w in (("cold", False), ("warm", True)):
    ms, hit, fa, opt = run(w)
    print("ext B=%d noise %.2f %s: %.3f ms/tick  %.0f QPs/s  warm hits %.3f  factorizations/QP %.2f  optimal %.4f"
          % (B, noise, name, ms, B / ms * 1e3, hit, fa, opt), flush=True)
