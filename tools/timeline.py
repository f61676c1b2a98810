"""dev tool: per-CTA and per-QP timeline of one step of the benchmark workload, from the measurement build (A1MPC_TIMELINE=1).

  python tools/timeline.py [--batch 1024] [--steps 20] [--lib PATH] [--json FILE]

Builds liba1mpc.so with -DA1MPC_TIMELINE=1 into a temporary directory (or loads --lib), runs bench.py's workload (config 2,
horizon 10) and, for --steps single steps after a warm-up, reads back what every class-kernel CTA recorded (%smid, %globaltimer
at entry and exit, QPs served) and every QP (start, end, factorisations).  Printed per class, for the step of median length:
CTAs with work, their start times (earliest, latest, how many started later than t0 + 20 us, t0 = the first CTA of the step to
start), SM time spent in CTAs that served no QP, the time from the last QP end to the class kernel's end, and the critical QP
(the one that ended last).  The instrumentation adds global stores and timer reads, so absolute times are those of the
measurement build; the library itself is built without it."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "a1-qp-mpc-controller_b200")
TL_CLASSES, TL_CTAS, TL_QPS = 8, 1024, 32768   # a1mpc_device.cuh, tl_cta / tl_qp
LATE_NS = 20000
NAMES = {1: "1-stance", 2: "trot (2-stance)", 3: "3-stance", 4: "4-stance", 5: "extended", 6: "compact schedules"}


def build_lib(tmp):
    lib = os.path.join(tmp, "liba1mpc_timeline.so")
    subprocess.check_call(["make", "-C", ROOT, "-s", "-j8", "OBJ=" + os.path.join(tmp, "obj"), "LIB=" + lib,
                           "EXTRA=-DA1MPC_TIMELINE=1", lib], stdout=subprocess.DEVNULL)
    return lib


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def analyse(buf):
    """buf: the u64 records of one step -> {class: metrics}, step length (ns)"""
    cta = buf[:TL_CLASSES * TL_CTAS * 4].reshape(TL_CLASSES, TL_CTAS, 4).astype(np.int64)
    qp = buf[TL_CLASSES * TL_CTAS * 4:].reshape(TL_CLASSES, TL_QPS, 4).astype(np.int64)
    qp[:, :, 2] = qp[:, :, 2] % 100 + qp[:, :, 2] // 100   # the iters output: interior-point + 100 x finisher factorisations
    ran = cta[:, :, 1] > 0
    t0 = cta[:, :, 1][ran].min()
    t_end = cta[:, :, 2][ran].max()
    out = {}
    for k in range(1, TL_CLASSES):
        if not ran[k].any():
            continue
        c = cta[k][ran[k]]
        bid = np.nonzero(ran[k])[0]
        work = c[:, 3] > 0
        q = qp[k]
        qv = q[:, 1] > 0
        m = {"ctas": int(len(c)), "ctas_with_work": int(work.sum()), "qps": int(qv.sum())}
        if work.any():
            st = c[work, 1] - t0
            m.update(first_start_us=st.min() / 1e3, last_start_us=st.max() / 1e3, late_ctas=int((st > LATE_NS).sum()),
                     kernel_end_us=(c[:, 2].max() - t0) / 1e3)
        m["empty_cta_sm_us"] = float((c[~work, 2] - c[~work, 1]).sum()) / 1e3
        m["empty_cta_max_us"] = float((c[~work, 2] - c[~work, 1]).max()) / 1e3 if (~work).any() else 0.0
        m["empty_cta_last_exit_us"] = float((c[~work, 2].max() - t0) / 1e3) if (~work).any() else 0.0
        if qv.any():
            idx = np.nonzero(qv)[0]
            last = idx[np.argmax(q[idx, 1])]
            m["last_qp_to_kernel_end_us"] = (c[:, 2].max() - q[last, 1]) / 1e3
            r3 = int(q[last, 3])
            m["critical_qp"] = {"q": int(last), "start_us": (q[last, 0] - t0) / 1e3, "end_us": (q[last, 1] - t0) / 1e3,
                                "length_us": (q[last, 1] - q[last, 0]) / 1e3, "factorizations": int(q[last, 2]),
                                "sm": r3 >> 32, "cta": (r3 >> 8) & 0xFFFFFF, "slot": r3 & 0xFF}
            m["qp_start_after_t0_plus_20us"] = int(((q[idx, 0] - t0) > LATE_NS).sum())
            m["factorizations_mean"] = float(q[idx, 2].mean())
        m["sms"] = int(len(np.unique(c[:, 0])))
        m["first_started_ctas"] = [int(b) for b in bid[np.argsort(c[:, 1])][:4]]
        out[k] = m
    return out, int(t_end - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--lib", default=None, help="a liba1mpc.so built with -DA1MPC_TIMELINE=1 (default: build one in a temporary directory)")
    ap.add_argument("--json", default=None, help="also write every step's metrics to this file")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="a1mpc_tl_")
    os.environ["A1MPC_LIB"] = args.lib or build_lib(tmp)
    sys.path.insert(0, PKG)
    import a1mpc
    lib = a1mpc.lib()
    if not hasattr(lib, "a1mpc_timeline_attach"):
        raise SystemExit("%s was not built with -DA1MPC_TIMELINE=1" % os.environ["A1MPC_LIB"])
    lib.a1mpc_timeline_attach.argtypes = [C.c_void_p, C.c_void_p]
    print("device:", device_line(), flush=True)

    B = args.batch
    eng = a1mpc.Engine(a1mpc.default_config(horizon=10), device=0)
    ring = []
    for r in range(8):   # bench.py's inputs (config 2, streams 0, 1, ...); the ring only has to keep the steps distinct
        d = a1mpc.DeviceBatch(eng, B, want_u=False, want_iters=False)
        d.upload(a1mpc.gen_states(B, 2, stream=r))
        ring.append(d)
    nwords = TL_CLASSES * (TL_CTAS + TL_QPS) * 4
    dbuf = eng.dalloc(nwords * 8)
    zeros = np.zeros(nwords, dtype=np.uint64)
    host = np.zeros(nwords, dtype=np.uint64)
    for i in range(args.warmup):
        eng.solve_ptrs(B, ring[i % 8].inp, ring[i % 8].out)
    eng.sync()
    a1mpc._check(lib.a1mpc_timeline_attach(eng.h, dbuf))
    steps = []
    for i in range(args.steps):
        a1mpc._check(lib.a1mpc_memcpy_h2d(eng.h, dbuf, zeros.ctypes.data, zeros.nbytes))
        eng.sync()
        eng.solve_ptrs(B, ring[i % 8].inp, ring[i % 8].out)
        eng.sync()
        a1mpc._check(lib.a1mpc_memcpy_d2h(eng.h, host.ctypes.data, dbuf, host.nbytes))
        eng.sync()
        steps.append(analyse(host))
    a1mpc._check(lib.a1mpc_timeline_attach(eng.h, None))

    lens = np.array([s[1] for s in steps])
    med = int(np.argsort(lens)[len(lens) // 2])
    print("B = %d, %d steps: first CTA start -> last CTA end %.1f us median (%.1f-%.1f)" % (B, len(lens), np.median(lens) / 1e3, lens.min() / 1e3, lens.max() / 1e3))
    print("step %d (median length %.1f us), t0 = first CTA start of the step:" % (med, lens[med] / 1e3))
    for k, m in steps[med][0].items():
        print("  class %d %s: %d CTAs on %d SMs, %d with work, %d QPs" % (k, NAMES.get(k, ""), m["ctas"], m["sms"], m["ctas_with_work"], m["qps"]))
        if "first_start_us" in m:
            print("    CTAs with work start %.1f .. %.1f us, %d after t0 + 20 us; kernel ends %.1f us" % (m["first_start_us"], m["last_start_us"], m["late_ctas"], m["kernel_end_us"]))
        print("    empty CTAs: %.1f SM-us in all, longest %.1f us, last exit at %.1f us" % (m["empty_cta_sm_us"], m["empty_cta_max_us"], m["empty_cta_last_exit_us"]))
        if "critical_qp" in m:
            cq = m["critical_qp"]
            print("    QPs started after t0 + 20 us: %d; last QP end -> kernel end %.1f us; factorizations/QP %.2f" % (m["qp_start_after_t0_plus_20us"], m["last_qp_to_kernel_end_us"], m["factorizations_mean"]))
            print("    critical QP %d: %.1f -> %.1f us (%.1f us, %d factorizations) on SM %d, CTA %d slot %d" % (cq["q"], cq["start_us"], cq["end_us"], cq["length_us"], cq["factorizations"], cq["sm"], cq["cta"], cq["slot"]))
    keys = ("late_ctas", "last_start_us", "empty_cta_sm_us", "last_qp_to_kernel_end_us", "kernel_end_us")
    print("medians over all %d steps:" % len(steps))
    for k in sorted({k for s in steps for k in s[0]}):
        vals = {key: np.median([s[0][k][key] for s in steps if k in s[0] and key in s[0][k]]) for key in keys if any(k in s[0] and key in s[0][k] for s in steps)}
        print("  class %d: %s" % (k, ", ".join("%s %.1f" % kv for kv in vals.items())))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": device_line(), "batch": B, "steps": [{"length_us": s[1] / 1e3, "classes": s[0]} for s in steps]}, f, indent=1, default=float)


if __name__ == "__main__":
    main()
