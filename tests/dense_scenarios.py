"""Dense-Hessian QPs with a different B_d per horizon step, for the suites of a1mpc_solve_dense_batch (tests/test_emu_dense.py on the
CPU emulator, tests/test_gpu_dense.py on the device).

ConvexMpc::calculate_qp_mats takes a B_mat_d_list, so a caller may give every step its own B_d (test/test_mpc.cpp:106-125).  The fused
solve does not take one; such callers build H, g with a1mpc_qp_mats_batch and solve them with a1mpc_solve_dense_batch.  Each family
here starts from the envelope families (tests/envelope_scenarios.py) and lets the body move through the horizon while the footholds
stay fixed in the world: at step k the body has moved by k steps of the commanded world velocity and turned by k steps of the
commanded yaw rate, so step k's B_d uses that step's trunk rotation and body-to-foot vectors.  B_d follows the reference's
calculate_B_mat_c and the forward-Euler discretisation (ConvexMpc.cpp:132-156), in numpy: the oracle's rollout computes one B_d per
call and would take seconds per batch; pin_rollout() pins these B_d, A_d, x0 and x_d to it.

The stance count is drawn uniformly before the mask, so the three- and four-foot classes are as common as the others.  At N = 20 the
dense path serves one and two feet; counts=(3, 4) gives the QPs it reports as unsupported.  Deterministic: numpy, seeded."""
import numpy as np

import envelope_scenarios as env

FAMILIES = env.FAMILIES
GRAVITY = -9.8
# floors on the oracle's optimum over each family's QPs, as fractions of the batch.  Measured on 256 QPs per family at N = 10: fz_max
# 0.32-0.80, vertex 0.51-0.73, edge 0.73-0.98, a whole foot at the vertex 0.20-0.36; on 64 QPs (one or two feet) at N = 20: fz_max
# 0.20-0.53, vertex 0.20-0.62, edge 0.81-0.98, foot at vertex 0.06-0.22
CENSUS_FLOORS = {10: dict(edge=0.6, vertex=0.35, foot0=0.1, fzmax=0.2), 20: dict(edge=0.6, vertex=0.12, foot0=0.03, fzmax=0.1)}
# floors on how much B_d moves from one step to the next, max_k |B_k - B_(k-1)| / |B_0| over the angular rows 6..8 of B_d: the median
# over a family (measured 1.7e-3 to 2.6e-3) and every single QP (measured at least 1.3e-4 over 8192 QPs), so the family cannot fall
# back to a constant B_d unnoticed
BD_STEP_MEDIAN = 1e-3
BD_STEP_MIN = 5e-5


def masks_with(ns):
    return [m for m in range(1, 16) if bin(m).count("1") == ns]


def draw_contact(rng, B, counts):
    """stance count uniform over `counts`, then the mask uniform among the masks with that count"""
    ns = rng.choice(np.asarray(counts), size=B)
    out = np.zeros(B, dtype=np.uint32)
    for c in counts:
        sel = np.nonzero(ns == c)[0]
        ms = np.asarray(masks_with(c), dtype=np.uint32)
        out[sel] = ms[rng.integers(0, len(ms), size=len(sel))]
    return out


def _rz(a):
    c, s, z, o = np.cos(a), np.sin(a), np.zeros_like(a), np.ones_like(a)
    return np.stack([np.stack([c, -s, z], -1), np.stack([s, c, z], -1), np.stack([z, z, o], -1)], -2)


def _skew(r):
    z = np.zeros(r.shape[:-1])
    x, y, w = r[..., 0], r[..., 1], r[..., 2]
    return np.stack([np.stack([z, -w, y], -1), np.stack([w, z, -x], -1), np.stack([-y, x, z], -1)], -2)


def b_d(cfg, R, foot):
    """calculate_B_mat_c + state_space_discretization: R [..,3,3] trunk rotation, foot [..,4,3] body-to-foot vectors in the world
    frame -> B_d [..,13,12]"""
    I = np.array(list(cfg.inertia)).reshape(3, 3)
    Iw_inv = np.linalg.inv(R @ I @ np.swapaxes(R, -1, -2))
    Bc = np.zeros(R.shape[:-2] + (13, 12))
    for leg in range(4):
        Bc[..., 6:9, 3 * leg:3 * leg + 3] = Iw_inv @ _skew(foot[..., leg, :])
        Bc[..., 9:12, 3 * leg:3 * leg + 3] = np.eye(3) / cfg.mass
    return Bc * cfg.dt


def step_pose(cfg, st, k):
    """trunk rotation [B,3,3] and body-to-foot vectors [B,4,3] at horizon step k: the body has moved by k dt v_d (world) and turned by
    k dt yaw_rate_d, the footholds are where they were at step 0"""
    B = st["x0"].shape[1]
    R = st["rot"].T.reshape(B, 3, 3)
    vdw = np.einsum("bij,jb->bi", R, st["ref"][5:8])
    Rk = _rz(k * cfg.dt * st["ref"][4]) @ R
    foot = st["foot"].T.reshape(B, 4, 3) - (k * cfg.dt * vdw)[:, None, :]
    return Rk, foot


def build(a1, cfg, name, B, seed, counts):
    """B QPs of family `name` at cfg.horizon with stance counts drawn from `counts`: the state dict `st` of the envelope family (its
    contact redrawn), A_d [B,13,13], B_list [B,13N,12] (per-step B_d), B_const [B,13N,12] (step 0's B_d at every step), x0 [B,13],
    x_d [B,13N] -- the arguments of ConvexMpc::calculate_qp_mats as compute_grf fills them (A1RobotControl.cpp:452-514)"""
    N, dt = cfg.horizon, cfg.dt
    st = env.family(a1, name, B, seed)
    rng = np.random.default_rng([seed, FAMILIES.index(name), N, 7])
    st["contact"] = draw_contact(rng, B, counts)
    e, p, w, v = st["x0"][0:3].T, st["x0"][3:6].T, st["x0"][6:9].T, st["x0"][9:12].T
    ref = st["ref"].T
    R = st["rot"].T.reshape(B, 3, 3)
    Ac = np.zeros((B, 13, 13))
    c, s = np.cos(e[:, 2]), np.sin(e[:, 2])
    Ac[:, 0, 6], Ac[:, 0, 7], Ac[:, 1, 6], Ac[:, 1, 7], Ac[:, 2, 8] = c, s, -s, c, 1.0
    Ac[:, 3:6, 9:12] = np.eye(3)
    Ac[:, 11, 12] = 1.0
    A_d = np.eye(13) + Ac * dt
    x0 = np.concatenate([e, p, w, v, np.full((B, 1), GRAVITY)], axis=1)
    vdw = np.einsum("bij,bj->bi", R, ref[:, 5:8])
    x_d = np.zeros((B, N, 13))
    for i in range(N):
        t = dt * (i + 1)
        x_d[:, i] = np.stack([ref[:, 0], ref[:, 1], e[:, 2] + ref[:, 4] * t, p[:, 0] + vdw[:, 0] * t, p[:, 1] + vdw[:, 1] * t, ref[:, 8],
                              ref[:, 2], ref[:, 3], ref[:, 4], vdw[:, 0], vdw[:, 1], np.zeros(B), np.full(B, GRAVITY)], axis=1)
    B_list = np.concatenate([b_d(cfg, *step_pose(cfg, st, k)) for k in range(N)], axis=1)
    B_const = np.tile(B_list[:, :13], (1, N, 1))
    return dict(st=st, contact=st["contact"], A_d=A_d, B_list=B_list, B_const=B_const, x0=x0, x_d=x_d.reshape(B, 13 * N))


def pin_rollout(O, ocfg, d, idx):
    """the numpy model against the oracle's rollout (pinned to the reference's calculate_qp_mats chain): A_d, x0 and x_d of the state
    itself, and step k's B_d as the rollout of a state posed at step k's rotation and footholds.  Returns the worst relative error."""
    st = d["st"]
    N = ocfg.horizon
    worst = 0.0
    for b in idx:
        one = {k: (v[b:b + 1].copy() if k == "contact" else v[:, b:b + 1].copy()) for k, v in st.items()}
        r = O.rollout(ocfg, O.Batch(one["x0"], one["rot"], one["foot"], one["ref"], one["contact"]), 0)
        worst = max(worst, np.abs(r["A_d"] - d["A_d"][b]).max(), np.abs(r["mpc_states"] - d["x0"][b]).max() / np.abs(d["x0"][b]).max(),
                    np.abs(r["mpc_states_d"] - d["x_d"][b]).max() / np.abs(d["x_d"][b]).max())
        for k in (1, N // 2, N - 1):
            Rk, fk = step_pose(ocfg, one, k)
            posed = O.Batch(one["x0"], Rk.reshape(1, 9).T.copy(), fk.reshape(1, 12).T.copy(), one["ref"], one["contact"])
            Bk = O.rollout(ocfg, posed, 0)["B_d_list"][:13]
            ours = d["B_list"][b, 13 * k:13 * k + 13]
            worst = max(worst, np.abs(Bk - ours).max() / np.abs(Bk).max())
    return worst


def qp_mats(O, ocfg, d, idx, key="B_list"):
    """the oracle's calculate_qp_mats on QPs idx: H [len,n,n], g [len,n]"""
    Hg = [O.qp_mats(ocfg, d["A_d"][b], d[key][b], d["x0"][b], d["x_d"][b]) for b in idx]
    return np.stack([h for h, _ in Hg]), np.stack([g for _, g in Hg])


def oracle_solve(O, ocfg, H, g, contact, nthreads=1):
    """O.solve_dense(MODE_EXACT) of every QP: u [B,n], certified [B] (info[1] == 1)"""
    from concurrent.futures import ThreadPoolExecutor

    def one(b):
        return O.solve_dense(ocfg, H[b], g[b], contact[b], O.MODE_EXACT)
    with ThreadPoolExecutor(max(1, nthreads)) as ex:
        res = list(ex.map(one, range(len(contact))))
    return np.stack([u for u, _ in res]), np.array([info[1] == 1 for _, info in res])


def bd_step(d):
    """per QP: max over k of |B_k - B_(k-1)|_max / |B_0|_max on the angular rows 6..8 of B_d"""
    B, N = d["B_list"].shape[0], d["B_list"].shape[1] // 13
    Bl = d["B_list"].reshape(B, N, 13, 12)[:, :, 6:9]
    return np.abs(np.diff(Bl, axis=1)).max(axis=(1, 2, 3)) / np.abs(Bl[:, 0]).max(axis=(1, 2))


def check_bd_step(name, d):
    s = bd_step(d)
    print("B_d step %-9s min %.2e  median %.2e  max %.2e" % (name, s.min(), np.median(s), s.max()))
    assert np.median(s) >= BD_STEP_MEDIAN and s.min() >= BD_STEP_MIN, (name, s.min(), np.median(s))


def class_counts(contact):
    ns = np.array([bin(int(c)).count("1") for c in contact])
    return {k: int((ns == k).sum()) for k in range(5)}


# Input contract of a1mpc_solve_dense_batch: the solver reads the upper triangle of H on the stance rows and columns and g on the stance
# rows only.  Each case edits one QP of a clean batch; "same" cases must give that QP's clean result bit for bit, "numerical" cases
# status NUMERICAL with u all zero, "no_contact" status NO_CONTACT with u all zero.
CASES = (("lower_nan", "same"), ("swing_nan", "same"), ("swing_inf", "same"), ("swing_huge", "same"),
         ("upper_nan", "numerical"), ("upper_inf", "numerical"), ("upper_huge", "numerical"), ("upper_far_nan", "numerical"),
         ("upper_far_ninf", "numerical"), ("diag_zero", "numerical"), ("diag_neg", "numerical"), ("diag_nan", "numerical"),
         ("diag_inf", "numerical"), ("diag_huge", "numerical"), ("g_nan", "numerical"), ("g_huge", "numerical"), ("no_contact", "no_contact"))


def stance_index(contact, N):
    """full indices (12 step + 3 leg + axis) of the stance variables, ascending"""
    legs = [leg for leg in range(4) if (int(contact) >> leg) & 1]
    return np.array(sorted(12 * s + 3 * leg + a for s in range(N) for leg in legs for a in range(3)), dtype=np.int64)


def edit(case, H, g, contact, N):
    """applies CASES entry `case` to one QP in place (H [n,n], g [n]); returns its contact mask"""
    n = 12 * N
    S = stance_index(contact, N)
    W = np.setdiff1d(np.arange(n), S)
    kind, _, what = case.rpartition("_")
    val = {"nan": np.nan, "inf": np.inf, "ninf": -np.inf, "huge": 1e300, "zero": 0.0, "neg": -1.0}.get(what)
    if case == "lower_nan":
        H[np.tril_indices(n, -1)] = np.nan
    elif kind == "swing":
        H[W, :] = val
        H[:, W] = val
        g[W] = val
    elif kind == "upper":
        H[S[0], S[5]] = val                  # the first stance row, a few columns along
    elif kind == "upper_far":
        H[S[1], S[-1]] = val                 # first step against the last
    elif kind == "diag":
        H[S[len(S) // 2], S[len(S) // 2]] = val
    elif kind == "g":
        g[S[-1]] = val
    elif case == "no_contact":
        return 0
    else:
        raise ValueError(case)
    return contact


def contract_plan(contact):
    """which QP each of CASES edits: [(qp, case, expect)].  The odd members of each stance class's queue, so that good and bad QPs
    alternate in each class; the swing cases go to QPs with a swing foot, and the cases rotate over the classes."""
    ns = np.array([bin(int(c)).count("1") for c in contact])
    free = {k: list(np.nonzero(ns == k)[0][1::2]) for k in range(1, 5)}
    plan = []
    for i, (case, expect) in enumerate(CASES):
        order = [1 + (i + j) % 4 for j in range(4)]
        if case.startswith("swing"):
            order = [k for k in order if k < 4]
        cls = next((k for k in order if free[k]), None)
        assert cls is not None, "the clean batch has too few QPs for the input-contract cases"
        plan.append((int(free[cls].pop(0)), case, expect))
    return plan


def contract_batch(H, g, contact, N):
    """copies of the clean batch with every case of contract_plan applied, and the plan"""
    H, g, contact = H.copy(), g.copy(), contact.copy()
    plan = contract_plan(contact)
    for b, case, _ in plan:
        contact[b] = edit(case, H[b], g[b], contact[b], N)
    return H, g, contact, plan


def check_contract(a1, u, status, u_clean, status_clean, labels):
    """the expectations of contract_batch's labels, and every QP it did not edit bit-identical to the clean call"""
    edited = {b for b, _, _ in labels}
    for b, case, expect in labels:
        if expect == "same":
            assert status[b] == status_clean[b] and np.array_equal(u[b], u_clean[b]), (case, b, status[b])
        else:
            want = a1.STATUS_NUMERICAL if expect == "numerical" else a1.STATUS_NO_CONTACT
            assert status[b] == want and np.array_equal(u[b], np.zeros_like(u[b])), (case, b, status[b], np.abs(u[b]).max())
    keep = np.array([b not in edited for b in range(len(status))])
    assert np.array_equal(status[keep], status_clean[keep]) and np.array_equal(u[keep], u_clean[keep])
