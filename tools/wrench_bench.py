"""dev tool: device time of the four-stance class kernel alone (all QPs of the batch have four stance feet), per launch, from the
library's per-class CUDA events (a1mpc_profile_begin / _end).  Runs the default weights and a q with a zero in q[6..11] (that
handle keeps the Ls form of the wrench-space solve; the default one uses the Hw^-1 + S form), at batch 1024 and 32768.
A1MPC_LIB selects the library, so two builds are compared by running this script once with each.  Prints one JSON line."""
import argparse, json, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "a1-qp-mpc-controller_b200"))
import a1mpc

Q_DEFAULT = list(a1mpc.default_config(horizon=10).q)
Q_ZERO = Q_DEFAULT[:6] + [0.0] + Q_DEFAULT[7:]   # no weight on the roll rate: Q0 singular


def run(N, B, q, K, W):
    eng = a1mpc.Engine(a1mpc.default_config(horizon=N, q=q))
    st = a1mpc.gen_states(B, 2, 777)
    st["contact"][:] = 15
    f, status, iters = eng.solve(st)
    d = a1mpc.DeviceBatch(eng, B, want_u=False, want_iters=False)
    d.upload(st)
    for _ in range(W):
        eng.solve_ptrs(B, d.inp, d.out)
    eng.sync()
    eng.profile_begin(K)
    for _ in range(K):
        eng.solve_ptrs(B, d.inp, d.out)
    eng.sync()
    class_ms, n = eng.profile_end()
    d.free()
    eng.close()
    fact = iters % 100 + iters // 100
    return {"N": N, "B": B, "q_zero": q != Q_DEFAULT, "ms_4stance": float(class_ms[3] / max(n, 1)), "launches": n,
            "status_hist": np.bincount(status, minlength=5).tolist(), "factorizations_mean": float(fact.mean()),
            "factorizations_p99": float(np.percentile(fact, 99))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--horizon", type=int, default=10)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rows = [run(a.horizon, B, q, a.steps if B <= 1024 else max(5, a.steps // 10), a.warmup) for B in (1024, 32768) for q in (Q_DEFAULT, Q_ZERO)]
    print(json.dumps({"lib": a1mpc.LIB_PATH, "gpu": gpu, "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
