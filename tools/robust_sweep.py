"""dev tool: status histogram over large synthetic batches (+ oracle spot check)"""
import os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200")); sys.path.insert(0, ROOT)
import a1mpc
from oracle import oracle_py as O
HW = dict(mass=13.5, inertia=[0.0178533, 0, 0, 0, 0.0377999, 0, 0, 0, 0.0456542], q=[150, 150, 50, 0, 0, 80, .2, .2, .2, .3, .3, .3, 0], r=[1e-2, 1e-2, 1e-3] * 4)
for N, wname, cid, B in ((10, "gazebo", 2, 524288), (10, "gazebo", 4, 524288), (10, "hardware", 4, 262144), (20, "gazebo", 2, 65536), (20, "gazebo", 4, 65536)):
    kw = HW if wname == "hardware" else {}
    eng = a1mpc.Engine(a1mpc.default_config(horizon=N, **kw))
    st = a1mpc.gen_states(B, cid, 12345)
    rng = np.random.default_rng(1)
    # sprinkle every stance pattern
    idx = rng.choice(B, B // 8, replace=False)
    st["contact"][idx] = rng.integers(1, 16, size=len(idx)).astype(np.uint32)
    t = time.time(); f, status, iters = eng.solve(st); dt = time.time() - t
    bad = np.nonzero(status != 0)[0]
    print("N=%d %s cid=%d B=%d: %.2fs status hist %s  ipm max %d rounds max %d" % (N, wname, cid, B, dt, np.bincount(status, minlength=5), (iters % 100).max(), (iters // 100).max()), flush=True)
    # every QP against the oracle, not a sample: round 1's 1 500 spot checks missed 1-in-70 000 certified-but-wrong answers
    nfull = B if N == 10 else min(B, 20000)
    chk = np.concatenate([bad[:20], np.arange(nfull)])
    sub = {k: (v[chk].copy() if k == "contact" else v[:, chk].copy()) for k, v in st.items()}
    ocfg = O.make_config(horizon=N, **({k: tuple(v) if isinstance(v, list) else v for k, v in kw.items()}))
    fo, info = O.compute_grf_batch(ocfg, O.Batch(sub["x0"], sub["rot"], sub["foot"], sub["ref"], sub["contact"]), O.MODE_EXACT, nthreads=O.hardware_threads())
    err = np.abs(f[:, chk] - fo).max(axis=0)
    e_all = err[len(bad[:20]):]; opt = status[:nfull] == 0
    print("   %d QPs against the oracle: max err of OPTIMAL %.2e, #(>1e-7) %d, #(>1e-4) %d (oracle verified %d/%d)   bad QPs: %s" % (nfull, e_all[opt].max(), int((e_all[opt] > 1e-7).sum()), int((e_all[opt] > 1e-4).sum()), int(info[:, 1].sum()), len(chk),
          [(int(b), int(status[b]), int(iters[b]), float(err[i])) for i, b in enumerate(bad[:20])]), flush=True)
    eng.close()
