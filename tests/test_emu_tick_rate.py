"""CPU: the kernels of the multi-rate tick (a1mpc_tick_set_mpc_period) on the block emulator.
  1. The masked pack kernels (pack_due_kernel, pack_ext_due_kernel, pack_ext2_due_kernel, warm_forget_no_contact_due_kernel) write, bit for
     bit, the records the unmasked kernels write for the due robots (as sets: the slot order follows the atomics) and the same outputs and
     warm words for them; every output word and warm word of the robots that are not due is untouched.
  2. tick_rate_kernel over many runs and every period 1..N: robot b solves on run n when n == 0 or n % period == b % period; j_b, the runs
     since its last solve, stays below the period; with a plan a robot that does not solve gets R^T u_j within 1e-13 of numpy, without one
     (HOLD) its forces stay; due robots' forces are never touched.  tick_rate_reset_kernel zeroes the masked robots' counters only.
  3. plan_forces_kernel: step 0 untouched, 1 <= step < N rotated plan step within 1e-13 of numpy, step >= N zero forces."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_tick_rate_py as E  # noqa: E402

B = 300          # three blocks, the last one partial
N = 10
TOL = 1e-13


def due_rule(n, period):
    b = np.arange(n.shape[0])
    return (n == 0) | (n % period == b % period)


def _bits(a):
    return a.view(np.uint64) if a.dtype == np.float64 else a


def _batch(rng, kind):
    st = dict(x0=rng.standard_normal((12, B)), rot=rng.standard_normal((9, B)), foot=rng.standard_normal((12, B)), ref=rng.standard_normal((9, B)),
              contact=rng.integers(0, 16, B).astype(np.uint32))
    sched = normals = None
    if kind > 0:
        sched = rng.integers(0, 16, (N, B)).astype(np.uint32)
        sched[:, rng.random(B) < 0.1] = 0                                        # robots without contact anywhere
        sched[:, rng.random(B) < 0.3] = np.array([9, 6] * (N // 2), np.uint32)[:, None]   # two feet in every step: queue 6 of pack_ext2
        normals = rng.standard_normal((12, B))
        normals[2::3] = np.abs(normals[2::3]) + 0.1
    return st, sched, normals


def _outputs(rng, want_u):
    return dict(f_body=rng.standard_normal((12, B)), status=rng.integers(-9, 9, B).astype(np.int32), iters=rng.integers(-9, 9, B).astype(np.int32),
                u_full=rng.standard_normal((12 * N, B)) if want_u else None)


def _records(kind, rec, count, S):
    """{queue: {b: record bits}} of what a pack kernel wrote"""
    out = {}
    if kind == 0:
        for ns in range(1, 5):
            r = rec[(ns - 1) * B:(ns - 1) * B + count[ns]].view(np.uint64)
            out[ns] = {int(x[42] & 0xffffffff): x.tobytes() for x in r}
    else:
        for q, base in ((5, 0), (6, B)):
            r = rec[base:base + count[q]].view(np.uint64)
            out[q] = {int(x[42] & 0xffffffff): x.tobytes() for x in r}
    return out


@pytest.mark.parametrize("want_u", [False, True], ids=["no_u", "u_full"])
@pytest.mark.parametrize("kind", [0, 1, 2], ids=["pack", "pack_ext", "pack_ext2"])
def test_masked_pack_matches_unmasked_pack_of_due_robots(kind, want_u):
    S = E.sizes()
    rd = S["rec"] if kind == 0 else S["rec_ext"]
    nrec = 4 * B if kind == 0 else 2 * B
    ww = S["warm_hdr"] + 4 * N
    rng = np.random.default_rng(10 * kind + want_u)
    checked = 0
    for period in (2, 3, 7, N):
        st, sched, normals = _batch(rng, kind)
        runs = rng.integers(0, 3 * period, B).astype(np.uint32)
        runs[rng.random(B) < 0.1] = 0
        due = due_rule(runs, period)
        outs0 = _outputs(rng, want_u)
        warm0 = rng.integers(1, 2**32, (B, ww), dtype=np.uint32) if kind > 0 else None
        res = []
        for masked in (False, True):
            rec = np.full((nrec, rd), np.nan)
            count = np.zeros(16, np.int32)
            outs = {k: (v.copy() if v is not None else None) for k, v in outs0.items()}
            warm = warm0.copy() if warm0 is not None else None
            E.pack(kind, N, st, sched, normals, runs if masked else None, period, rec, B, count, outs, warm)
            res.append((_records(kind, rec, count, S), outs, warm))
        (full, outs_full, warm_full), (part, outs_part, warm_part) = res
        for q in full:
            want = {b: r for b, r in full[q].items() if due[b]}
            assert part[q] == want, (period, q)
            checked += len(want)
        for k, v0 in outs0.items():
            if v0 is None:
                continue
            assert np.array_equal(_bits(outs_part[k])[..., ~due], _bits(v0)[..., ~due]), (period, k)     # skipped robots: untouched
            assert np.array_equal(_bits(outs_part[k])[..., due], _bits(outs_full[k])[..., due]), (period, k)
        if warm0 is not None:
            assert np.array_equal(warm_part[~due], warm0[~due]) and np.array_equal(warm_part[due], warm_full[due]), period
            assert (warm_full[:, 0] != warm0[:, 0]).any()     # the unmasked kernel did clear some slots
        assert (~due).sum() > 0.3 * B
    assert checked > 0.5 * B


def _restated_plan_forces(rot, plan, j):
    """numpy: f[3 leg + a] = sum_k R[k][a] u[12 j + 3 leg + k], R row-major [9][B]"""
    b = np.arange(rot.shape[1])
    R = rot.reshape(3, 3, -1)
    u = plan.reshape(N, 4, 3, -1)[np.minimum(j, N - 1), :, :, b]        # [B, 4, 3]
    f = np.einsum("kab,blk->lab", R, u)                                   # [4, 3, B]
    return f.reshape(12, -1)


@pytest.mark.parametrize("playback", ["hold", "plan"])
def test_counters_and_playback_over_many_runs(playback):
    rng = np.random.default_rng(5 if playback == "plan" else 6)
    worst = 0.0
    for period in range(1, N + 1):
        runs, since = np.zeros(B, np.uint32), np.zeros(B, np.uint32)
        n = 0
        last = np.full(B, -1)
        for _ in range(3 * period + 25):
            rot = rng.standard_normal((9, B))
            plan = rng.standard_normal((12 * N, B)) if playback == "plan" else None
            f0 = rng.standard_normal((12, B))
            f = f0.copy()
            E.tick_rate(B, period, N, runs, since, rot, plan, f)
            due = due_rule(np.full(B, n), period)
            last = np.where(due, n, last)
            j = n - last
            assert np.array_equal(since, j.astype(np.uint32)), (period, n)
            assert (j <= period - 1).all() and (j < N).all()
            assert np.array_equal(_bits(f[:, due]), _bits(f0[:, due]))
            if playback == "plan":
                want = _restated_plan_forces(rot, plan, j)
                if (~due).any():
                    worst = max(worst, float(np.abs(f[:, ~due] - want[:, ~due]).max()))
            else:
                assert np.array_equal(_bits(f), _bits(f0))
            n += 1
        assert due_rule(runs, period).tolist() == due_rule(np.full(B, n), period).tolist()   # the stored counter keeps the rule
    assert worst <= TOL, worst


def test_reset_kernel_zeroes_masked_counters_only():
    rng = np.random.default_rng(8)
    runs0, since0 = rng.integers(1, 40, B).astype(np.uint32), rng.integers(1, 9, B).astype(np.uint32)
    for mask in (np.zeros(B, np.uint8), np.ones(B, np.uint8), ((rng.random(B) < 0.25) * rng.integers(1, 256, B)).astype(np.uint8)):
        runs, since = runs0.copy(), since0.copy()
        E.tick_rate_reset(B, mask, runs, since)
        m = mask != 0
        assert (runs[m] == 0).all() and (since[m] == 0).all()
        assert np.array_equal(runs[~m], runs0[~m]) and np.array_equal(since[~m], since0[~m])


def test_plan_forces_kernel():
    rng = np.random.default_rng(9)
    rot, plan, f0 = rng.standard_normal((9, B)), rng.standard_normal((12 * N, B)), rng.standard_normal((12, B))
    step = rng.integers(0, N + 3, B).astype(np.uint32)
    step[:20] = 0
    step[20:40] = N
    step[40:45] = 2**32 - 1
    f = f0.copy()
    E.plan_forces(B, N, rot, plan, step, f)
    zero, past = step == 0, step >= N
    mid = ~zero & ~past
    assert np.array_equal(_bits(f[:, zero]), _bits(f0[:, zero]))
    assert (f[:, past] == 0.0).all()
    want = _restated_plan_forces(rot, plan, step.astype(np.int64))
    assert np.abs(f[:, mid] - want[:, mid]).max() <= TOL
    assert mid.sum() > 0.5 * B
