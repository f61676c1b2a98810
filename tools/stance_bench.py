"""dev tool: device time of the QP-branch stance controller (a1mpc_stance_qp_batch) on device pointers.

  python tools/stance_bench.py [--sizes 1024,16384,65536] [--repeats 5] [--iters 50] [--ticks 20] [--json PATH]

For each batch size, with the card's name and power limit read (nvidia-smi, read-only query) in the same run:
  (a) a1mpc_stance_qp_batch: PD law + QP from the controller state, batch-major arrays;
  (b) a1mpc_grf_qp_batch on QP-major device arrays precomputed from (a)'s own root_acc: the solve-only floor;
  (c) one QP-mode control tick chained on device pointers: leg kinematics -> update_plan -> swing legs -> stance QP -> joint torques.
(a) and (b) alternate over the repeats; each repeat is `iters` calls between two CUDA events on the handle's stream after a warm-up.
Reports min / median / max ms per call and M robots/s, and the share of OPTIMAL robots.  Inputs: tests/stance_scenarios.py (gazebo
QP gains, all 16 contact masks).  Not part of bench.py's contract."""
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
from stance_scenarios import gains, robots

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


def stats(ms, B):
    ms = np.array(ms)
    return dict(ms_min=float(ms.min()), ms_median=float(np.median(ms)), ms_max=float(ms.max()),
                mrobots_per_s_median=float(B / np.median(ms) / 1e3), mrobots_per_s_range=[float(B / ms.max() / 1e3), float(B / ms.min() / 1e3)])


def bench_size(eng, B, repeats, iters, ticks, ptrs_to_free):
    L = a1mpc.lib()
    mass, kdl, kpa, kda = gains("gazebo")
    st = robots(B, 2026 + B, "gazebo")
    d = {k: upload(eng, st[k]) for k in FIELDS}
    d_f, d_s, d_acc = eng.dalloc(12 * B * 8), eng.dalloc(B * 4), eng.dalloc(6 * B * 8)
    ptrs_to_free += list(d.values()) + [d_f, d_s, d_acc]
    g = [v.ctypes.data for v in (kdl, kpa, kda)]

    def stance(acc=None):
        a1mpc._check(L.a1mpc_stance_qp_batch(eng.h, B, C.c_size_t(B), d["x0"], d["rot"], d["rot_z"], d["foot"], d["contact"], d["des"], d["kp_linear"],
                                             *g, d_f, d_s, acc))
    stance(d_acc)
    eng.sync()
    acc = np.zeros((6, B)); status = np.zeros(B, dtype=np.int32)
    a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, acc.ctypes.data, d_acc, acc.nbytes))
    a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, status.ctypes.data, d_s, status.nbytes))
    eng.sync()
    stance_mask = (st["contact"] & 15) != 0
    share = float((status[stance_mask] == a1mpc.STATUS_OPTIMAL).mean())
    # (b): the QP alone on QP-major device arrays of the same robots
    qm = {k: upload(eng, np.ascontiguousarray(v.T)) for k, v in (("acc", acc), ("rot_z", st["rot_z"]), ("rot", st["rot"]), ("foot", st["foot"]))}
    q_f, q_s = eng.dalloc(12 * B * 8), eng.dalloc(B * 4)
    ptrs_to_free += list(qm.values()) + [q_f, q_s]

    def grf():
        a1mpc._check(L.a1mpc_grf_qp_batch(eng.h, B, qm["acc"], qm["rot_z"], qm["rot"], qm["foot"], d["contact"], q_f, q_s))
    grf()
    eng.sync()
    fg, sg = np.zeros((B, 12)), np.zeros(B, dtype=np.int32)
    f = np.zeros((12, B))
    a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, fg.ctypes.data, q_f, fg.nbytes)); a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, sg.ctypes.data, q_s, sg.nbytes))
    a1mpc._check(L.a1mpc_memcpy_d2h(eng.h, f.ctypes.data, d_f, f.nbytes))
    eng.sync()
    same = bool(np.array_equal(fg.T, f) and np.array_equal(sg, status))
    for _ in range(3):   # warm-up of both shapes
        stance(); grf()
    eng.sync()
    ta, tb = [], []
    for _ in range(repeats):
        ta.append(timed(eng, stance, iters))
        tb.append(timed(eng, grf, iters))
    # (c): the QP-mode tick chain
    rng = np.random.default_rng(B)
    rho_fix = np.array([[0.1805, 0.047, 0.0838, 0.21, 0.21], [0.1805, -0.047, -0.0838, 0.21, 0.21],
                        [-0.1805, 0.047, 0.0838, 0.21, 0.21], [-0.1805, -0.047, -0.0838, 0.21, 0.21]]).reshape(20)
    rho_opt = np.zeros(12)
    T = ticks
    q = np.tile(np.array([0.0, 0.8, -1.6] * 4)[None, :, None], (T, 1, B)) + 0.05 * rng.standard_normal((T, 12, B))
    d_q, d_force = upload(eng, q), upload(eng, rng.uniform(0.0, 80.0, (T, 4, B)))
    d_mode, d_gc = upload(eng, np.ones(B, dtype=np.uint32)), upload(eng, np.zeros((4, B)))
    d_sp = upload(eng, np.repeat(rng.choice([2.0, 3.0, 4.0], B)[None, :], 4, axis=0))
    d_lv, d_lvd, d_pos = upload(eng, st["x0"][9:12]), upload(eng, st["des"][6:9]), upload(eng, st["x0"][3:6])
    d_plan, d_trel, d_jac, d_fk, d_con = eng.dalloc(B * 4), eng.dalloc(12 * B * 8), eng.dalloc(36 * B * 8), eng.dalloc(12 * B * 8), eng.dalloc(B * 4)
    d_tau = upload(eng, np.zeros((12, B)))
    sw = eng.swing_alloc(B)
    ptrs_to_free += [d_q, d_force, d_mode, d_gc, d_sp, d_lv, d_lvd, d_pos, d_plan, d_trel, d_jac, d_fk, d_con, d_tau, sw]
    gp = a1mpc.default_gait_params(10)
    kp, kd = np.array([300.0, 400, 400] * 4), np.array([8.0, 8, 8] * 4)
    km, tg = np.array([0.1, 0.1, 0.04]), np.array([0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0])
    tick_no = [0]

    def tick():
        t = tick_no[0] % T
        tick_no[0] += 1
        a1mpc._check(L.a1mpc_leg_kinematics_batch(eng.h, B, C.c_void_p(d_q.value + t * 12 * B * 8), None, d["rot"], rho_opt.ctypes.data, rho_fix.ctypes.data,
                                                  None, d_jac, None, d["foot"], None))
        a1mpc._check(L.a1mpc_update_plan_batch(eng.h, B, C.byref(gp), d_gc, d_sp, d_mode, d_lv, d_lvd, d["rot_z"], d["rot"], d_pos, d_plan, None, d_trel,
                                               None, None))
        a1mpc._check(L.a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), kp.ctypes.data, kd.ctypes.data, sw, 0.0025, d_gc, d_plan, d["rot_z"], d["foot"],
                                              d_trel, C.c_void_p(d_force.value + t * 4 * B * 8), d_fk, d_con, None, None))
        a1mpc._check(L.a1mpc_stance_qp_batch(eng.h, B, C.c_size_t(B), d["x0"], d["rot"], d["rot_z"], d["foot"], d_con, d["des"], d["kp_linear"], *g,
                                             d_f, d_s, None))
        a1mpc._check(L.a1mpc_joint_torques_batch(eng.h, B, d_f, d_fk, d_jac, d_con, km.ctypes.data, tg.ctypes.data, d_tau))
    for _ in range(T):
        tick()
    eng.sync()
    tc = [timed(eng, tick, T) for _ in range(repeats)]
    return dict(B=B, optimal_share=share, grf_bit_identical=same, stance_qp=stats(ta, B), grf_qp_floor=stats(tb, B), qp_mode_tick=stats(tc, B))


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
    eng = a1mpc.Engine(a1mpc.default_config(mass=gains("gazebo")[0]))
    rec = dict(device=dev, repeats=a.repeats, iters=a.iters, results=[])
    ptrs = []
    for B in [int(s) for s in a.sizes.split(",")]:
        r = bench_size(eng, B, a.repeats, a.iters, a.ticks, ptrs)
        rec["results"].append(r)
        print("B=%6d  stance_qp %.3f ms [%.3f-%.3f] %.2f M/s | grf_qp floor %.3f ms [%.3f-%.3f] %.2f M/s | QP-mode tick %.3f ms [%.3f-%.3f] | OPTIMAL %.2f %% | "
              "bit-identical to grf_qp %s" % (B, r["stance_qp"]["ms_median"], r["stance_qp"]["ms_min"], r["stance_qp"]["ms_max"],
                                              r["stance_qp"]["mrobots_per_s_median"], r["grf_qp_floor"]["ms_median"], r["grf_qp_floor"]["ms_min"],
                                              r["grf_qp_floor"]["ms_max"], r["grf_qp_floor"]["mrobots_per_s_median"], r["qp_mode_tick"]["ms_median"],
                                              r["qp_mode_tick"]["ms_min"], r["qp_mode_tick"]["ms_max"], 100 * r["optimal_share"], r["grf_bit_identical"]),
              flush=True)
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
