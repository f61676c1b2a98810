"""GPU: a1mpc_tick_reset_robots on the inputs of tick_scenarios.tick_inputs.  The core check: tick A runs a standstill-then-walking run, its
masked robots are reset mid-run, and from then on every output of every tick is bit-identical to a tick F created at the moment of the reset
(for the masked robots) and to a tick U that never saw the reset (for the others).  So a reset robot starts over exactly as a fresh tick does,
and no other robot notices: the gait counters, swing filters, IMU filters, command state, EKF and warm-start faces of the batch stay per robot.
Also: repeated overlapping resets, all-one mask = a1mpc_tick_reset, all-zero mask = no call, host mask = device mask, resets before the first
run, two partial resets before one run, a partial reset superseded by a full one, a 1 % reset at B = 65 536, and argument errors."""
import ctypes as C

import numpy as np
import pytest

from command_scenarios import DT
from tick_scenarios import OUT_SPECS, DeviceSeqs, d2h, first_difference, h2d, tick_inputs

pytestmark = pytest.mark.gpu

FULL = "full"   # a resets entry: a1mpc_tick_reset instead of a mask


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def engines(a1):
    es = {N: a1.Engine(a1.default_config(horizon=N)) for N in (10, 20)}
    yield es
    for e in es.values():
        e.close()


def _params(a1, variant, kind, N):
    """kind: qp, held (MPC, gait.horizon 0) or sched (MPC, gait.horizon N)"""
    tp = a1.default_tick_params(variant, a1.TICK_QP if kind == "qp" else a1.TICK_MPC)
    if kind == "sched":
        tp.gait.horizon = N
    return tp


def _run(a1, eng, tp, ds, B, T, t0=0, resets=None, host_masks=False):
    """ticks t0 .. T-1 of a tick created before tick t0, on device pointers.  resets {t: [mask or FULL, ...]} are applied in order before
    tick t: a mask through reset_robots (host array) or reset_robots_ptr (device copy), FULL through reset().  Returns {t: host outputs}."""
    L = a1.lib()
    resets = resets or {}
    mpc = tp.mode == a1.TICK_MPC
    keys = [k for k in OUT_SPECS if mpc or k != "ref"]
    d = {k: eng.dalloc(int(np.prod(OUT_SPECS[k][0] + (B,))) * np.dtype(OUT_SPECS[k][1]).itemsize) for k in keys}
    outs = a1.TickOutputs(*[d.get(k) for k in a1.TICK_OUTPUTS])
    dmasks = []
    tick = a1.Tick(eng, B, tp)
    res = {}
    try:
        for t in range(t0, T):
            for m in resets.get(t, ()):
                if isinstance(m, str):
                    tick.reset()
                elif host_masks:
                    tick.reset_robots(m)
                else:
                    p = eng.dalloc(B)
                    dmasks.append(p)
                    h2d(a1, eng, p, np.ascontiguousarray(m, dtype=np.uint8))
                    tick.reset_robots_ptr(p.value)
            ins = a1.TickInputs(*[(ds.speed if k == "gait_counter_speed" else ds.at(k, t)) for k in a1.TICK_INPUTS])
            tick.run_ptrs(DT, ins, outs)
            res[t] = {k: d2h(a1, eng, d[k], OUT_SPECS[k][0] + (B,), OUT_SPECS[k][1]) for k in keys}
    finally:
        tick.close()
        for p in list(d.values()) + dmasks:
            L.a1mpc_device_free(eng.h, p)
    return res


def _expected(starts, runs, B, ts):
    """per tick t in ts, the outputs robot b must have: those of runs[s] for the latest start s <= t whose robots include b.  starts is
    a list of (tick, bool mask) with runs[tick] the fresh tick created there (tick 0: the tick that never saw a reset)"""
    want = {}
    for t in ts:
        src = np.zeros(B, dtype=np.int64)
        for s, m in starts:
            if s <= t:
                src[m] = s
        want[t] = {}
        for k, v in runs[0][t].items():
            out = v.copy()
            for s, _ in starts:
                if 0 < s <= t:
                    sel = src == s
                    out[..., sel] = runs[s][t][k][..., sel]
            want[t][k] = out
    return want


def _diff(got, want):
    ts = sorted(want)
    return first_difference([got[t] for t in ts], [want[t] for t in ts])


def _check_resets(a1, eng, tp, B, T, events, seed):
    """tick A with the partial resets of `events` {t: mask} against a fresh tick per event and one that never saw a reset"""
    seqs, speed = tick_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        got = _run(a1, eng, tp, ds, B, T, resets={t: [m] for t, m in events.items()})
        runs = {0: _run(a1, eng, tp, ds, B, T)}
        for t in events:
            runs[t] = _run(a1, eng, tp, ds, B, T, t0=t)
    finally:
        ds.free()
    first = min(events)
    want = _expected([(0, np.ones(B, bool))] + [(t, m != 0) for t, m in sorted(events.items())], runs, B, range(first, T))
    return got, want, runs[0]


def _status_counts(res):
    return [dict(zip(*np.unique(r["status"], return_counts=True))) for r in res.values()]


CASES = [(v, kind, 10) for v in (0, 1, 2) for kind in ("qp", "held", "sched")] + [(0, "held", 20), (0, "sched", 20)]


@pytest.mark.parametrize("variant,kind,N", CASES, ids=["v%d-%s-n%d" % c for c in CASES])
def test_reset_robots_matches_fresh_and_untouched_ticks(a1, engines, variant, kind, N):
    # tick 66: walking since tick 5, half toggled out at 18 and a quarter at 24, so the masked robots are caught walking and standing,
    # mid-swing and in contact, with the IMU windows and the 60-sample recent-contact windows full
    B, T, R = 512, 74, 66
    rng = np.random.default_rng(1000 + 10 * variant + N)
    mask = (rng.random(B) < 0.25).astype(np.uint8)
    got, want, untouched = _check_resets(a1, engines[N], _params(a1, variant, kind, N), B, T, {R: mask}, seed=40 + variant)
    assert _diff(got, want) is None, _diff(got, want)
    # the reset is visible: a masked robot's outputs leave the run it would have had
    m = mask != 0
    assert any(not np.array_equal(got[t]["tau"][:, m], untouched[t]["tau"][:, m]) for t in range(R, T))


def test_repeated_overlapping_resets(a1, engines):
    B, T = 384, 60
    rng = np.random.default_rng(5)
    a = rng.random(B) < 0.3
    b = (rng.random(B) < 0.3) | (a & (rng.random(B) < 0.5))   # overlaps a
    c = (rng.random(B) < 0.3) | (b & (rng.random(B) < 0.5))   # overlaps b
    events = {20: a.astype(np.uint8), 35: b.astype(np.uint8), 48: c.astype(np.uint8)}
    for kind in ("held", "sched"):
        got, want, _ = _check_resets(a1, engines[10], _params(a1, 0, kind, 10), B, T, events, seed=61)
        assert _diff(got, want) is None, (kind, _diff(got, want))


def _mode_runs(a1, eng, tp, B, T, seed, variants):
    seqs, speed = tick_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        return [_run(a1, eng, tp, ds, B, T, **kw) for kw in variants]
    finally:
        ds.free()


@pytest.mark.parametrize("kind", ["qp", "held", "sched"])
def test_all_one_mask_is_reset_and_all_zero_mask_is_no_call(a1, engines, kind):
    B, T, R = 256, 40, 30
    tp = _params(a1, 2, kind, 10)
    ones, zeros = np.ones(B, np.uint8), np.zeros(B, np.uint8)
    full, ones_r, plain, zeros_r = _mode_runs(a1, engines[10], tp, B, T, 8, [dict(resets={R: [FULL]}), dict(resets={R: [ones]}), {},
                                                                             dict(resets={R: [zeros], R + 3: [zeros, zeros]})])
    assert _diff(ones_r, full) is None, _diff(ones_r, full)
    assert _diff(zeros_r, plain) is None, _diff(zeros_r, plain)


def test_host_mask_matches_device_mask(a1, engines):
    B, T, R = 256, 36, 28
    rng = np.random.default_rng(3)
    m8 = ((rng.random(B) < 0.4) * rng.integers(1, 256, B)).astype(np.uint8)   # any nonzero byte marks a robot
    mb = m8 != 0
    tp = _params(a1, 0, "held", 10)
    dev, host_u8, host_bool = _mode_runs(a1, engines[10], tp, B, T, 12, [dict(resets={R: [m8]}), dict(resets={R: [m8]}, host_masks=True),
                                                                          dict(resets={R: [mb]}, host_masks=True)])
    assert _diff(host_u8, dev) is None and _diff(host_bool, dev) is None


def test_reset_orders(a1, engines):
    """a partial reset before the first run; two partial resets before one run (their union); a partial reset then a full one"""
    B, T, R = 256, 40, 26
    rng = np.random.default_rng(4)
    a, b = rng.random(B) < 0.3, rng.random(B) < 0.3
    tp = _params(a1, 0, "sched", 10)
    plain, before_first, union, one, superseded, full = _mode_runs(
        a1, engines[10], tp, B, T, 14,
        [{}, dict(resets={0: [a.astype(np.uint8)]}), dict(resets={R: [a.astype(np.uint8), b.astype(np.uint8)]}),
         dict(resets={R: [(a | b).astype(np.uint8)]}), dict(resets={R: [a.astype(np.uint8), FULL]}), dict(resets={R: [FULL]})])
    assert _diff(before_first, plain) is None, _diff(before_first, plain)
    assert _diff(union, one) is None, _diff(union, one)
    assert _diff(superseded, full) is None, _diff(superseded, full)


def test_large_batch_one_percent(a1, engines):
    B, T, R = 65536, 7, 4
    rng = np.random.default_rng(9)
    mask = (rng.random(B) < 0.01).astype(np.uint8)
    got, want, _ = _check_resets(a1, engines[10], _params(a1, 0, "held", 10), B, T, {R: mask}, seed=21)
    assert _diff(got, want) is None, _diff(got, want)
    print("B=%d, %d robots reset before tick %d: status counts of ticks %d-%d %s" % (B, int(mask.sum()), R, R, T - 1,
                                                                                   _status_counts({t: got[t] for t in range(R, T)})))


def test_argument_errors_on_a_live_tick(a1, engines):
    L = a1.lib()
    B = 64
    tick = a1.Tick(engines[10], B, _params(a1, 0, "held", 10))
    try:
        assert L.a1mpc_tick_reset_robots(tick.t, None) == -1 and b"null argument" in L.a1mpc_last_error()
        for bad in (np.ones(B + 1, bool), np.ones(B, np.int32), np.ones((2, B), bool)):
            with pytest.raises(ValueError):
                tick.reset_robots(bad)
        # the tick still runs after the rejected calls
        seqs, speed = tick_inputs(B, 2, 2)
        tick.reset_robots(np.ones(B, bool))
        tau, _ = tick.run(DT, *(seqs[n][0] for n in a1.TICK_INPUTS[:-1]), speed)
        assert np.isfinite(tau).all()
    finally:
        tick.close()
