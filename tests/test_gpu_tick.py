"""GPU tests of the whole-tick call (a1mpc_tick_*): every output of every tick bit-identical to the hand-built chain of the staged entry
points on the same inputs (tests/tick_scenarios.py, the chain of test_gpu_command.py's closed loops, which is checked against the oracle
there), in both stance modes and for the three adapter variants; host and device arrays; reset; the cold solve at horizon 20; a large batch;
argument errors on a live handle."""
import ctypes as C

import numpy as np
import pytest

from command_scenarios import DT
from tick_scenarios import DeviceSeqs, first_difference, staged_chain, tick_inputs, tick_run_device

pytestmark = pytest.mark.gpu

VARIANTS = dict(gazebo=0, hardware=1, isaac=2)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def eng(a1):
    e = a1.Engine(a1.default_config(horizon=10))
    yield e
    e.close()


def _compare(a1, eng, tp, B, T, seed):
    seqs, speed = tick_inputs(B, T, seed)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    try:
        want = staged_chain(a1, eng, tp, ds, B, T, DT)
        tick = a1.Tick(eng, B, tp)
        try:
            got = tick_run_device(a1, eng, tick, ds, B, T, DT)
        finally:
            tick.close()
    finally:
        ds.free()
    return got, want


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("mode", ["mpc", "qp"])
def test_tick_bit_identical_to_staged_chain(a1, eng, variant, mode):
    B, T = 1024, 30
    tp = a1.default_tick_params(VARIANTS[variant], a1.TICK_MPC if mode == "mpc" else a1.TICK_QP)
    got, want = _compare(a1, eng, tp, B, T, seed=41 + VARIANTS[variant])
    assert first_difference(got, want) is None, first_difference(got, want)
    modes = np.array([g["movement_mode"] for g in got])
    assert modes[:5].sum() == 0 and modes[5:].sum() > 0 and (modes[-1] == 0).any()     # standstill, walking, toggled out
    print("%s %s: %d ticks bit-identical, last tick status %s" % (variant, mode, T, np.bincount(got[-1]["status"], minlength=5)))


def test_host_and_device_arrays_agree(a1, eng):
    B, T = 256, 8
    tp = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC)
    seqs, speed = tick_inputs(B, T, 7)
    ds = DeviceSeqs(a1, eng, seqs, speed)
    tick = a1.Tick(eng, B, tp)
    try:
        dev = tick_run_device(a1, eng, tick, ds, B, T, DT)
        tick.reset()
        host = []
        for t in range(T):
            tau, o = tick.run(DT, *(seqs[k][t] for k in a1.TICK_INPUTS[:-1]), speed)
            o["tau"] = tau
            host.append(o)
    finally:
        tick.close()
        ds.free()
    assert first_difference(host, dev) is None, first_difference(host, dev)


def test_reset_reproduces_the_first_ticks(a1, eng):
    B, T = 512, 12
    for mode in (a1.TICK_MPC, a1.TICK_QP):
        tp = a1.default_tick_params(a1.VARIANT_ISAAC, mode)
        seqs, speed = tick_inputs(B, T, 3)
        ds = DeviceSeqs(a1, eng, seqs, speed)
        tick = a1.Tick(eng, B, tp)
        try:
            first = tick_run_device(a1, eng, tick, ds, B, T, DT)
            tick.reset()
            again = tick_run_device(a1, eng, tick, ds, B, T, DT)
        finally:
            tick.close()
            ds.free()
        assert first_difference(again, first) is None, (mode, first_difference(again, first))


def test_horizon_20_cold_solve(a1):
    e = a1.Engine(a1.default_config(horizon=20))
    try:
        tp = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC)
        got, want = _compare(a1, e, tp, 256, 2, seed=5)
    finally:
        e.close()
    assert first_difference(got, want) is None, first_difference(got, want)
    assert (got[-1]["status"] == a1.STATUS_OPTIMAL).mean() > 0.99, np.bincount(got[-1]["status"])


@pytest.mark.parametrize("mode", ["mpc", "qp"])
def test_large_batch_bit_identical(a1, eng, mode):
    B, T = 65536, 3
    tp = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_MPC if mode == "mpc" else a1.TICK_QP)
    got, want = _compare(a1, eng, tp, B, T, seed=11)
    assert first_difference(got, want) is None, first_difference(got, want)
    print("B=%d %s: status counts per tick %s" % (B, mode, [np.bincount(g["status"], minlength=5).tolist() for g in got]))


def test_argument_errors(a1, eng):
    L = a1.lib()
    B = 64
    tp = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP)
    t = C.c_void_p()
    e32 = a1.Engine(a1.default_config(precision=32))
    try:
        assert L.a1mpc_tick_create(e32.h, B, C.byref(tp), C.byref(t)) == -1 and b"precision" in L.a1mpc_last_error()
    finally:
        e32.close()
    for bad in (dict(mode=2), dict(variant=3), dict(cps=0.0)):
        p = a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP)
        if "mode" in bad:
            p.mode = bad["mode"]
        if "variant" in bad:
            p.command.variant = bad["variant"]
        if "cps" in bad:
            p.gait.counter_per_swing = bad["cps"]
        assert L.a1mpc_tick_create(eng.h, B, C.byref(p), C.byref(t)) == -1, bad
    assert L.a1mpc_tick_create(eng.h, 0, C.byref(tp), C.byref(t)) == -1
    seqs, speed = tick_inputs(B, 1, 1)
    host = {k: np.ascontiguousarray(seqs[k][0]) for k in a1.TICK_INPUTS[:-1]}
    host["gait_counter_speed"] = speed
    tick = a1.Tick(eng, B, tp)
    dtau = eng.dalloc(12 * B * 8)
    try:
        ins = a1.TickInputs(*[host[k].ctypes.data for k in a1.TICK_INPUTS])
        tau, ref = np.zeros((12, B)), np.zeros((9, B))
        ok = a1.TickOutputs(tau.ctypes.data, None, None, None, None, None, None)
        tick.run_ptrs(DT, ins, ok)
        for dt in (0.0, -DT):
            with pytest.raises(a1.A1MpcError, match="dt"):
                tick.run_ptrs(dt, ins, ok)
        with pytest.raises(a1.A1MpcError, match="ref"):
            tick.run_ptrs(DT, ins, a1.TickOutputs(tau.ctypes.data, None, None, None, None, None, ref.ctypes.data))
        with pytest.raises(a1.A1MpcError, match="all-host or all-device"):
            tick.run_ptrs(DT, ins, a1.TickOutputs(dtau, None, None, None, None, None, None))
        with pytest.raises(a1.A1MpcError, match="null"):
            tick.run_ptrs(DT, ins, a1.TickOutputs())
        tick.run_ptrs(DT, ins, ok)   # the handle and the tick still work after the rejected calls
        assert np.isfinite(tau).all()
    finally:
        L.a1mpc_device_free(eng.h, dtau)
        tick.close()


def test_engine_close_destroys_its_ticks_first(a1):
    e = a1.Engine(a1.default_config())
    B = 64
    tick = a1.Tick(e, B, a1.default_tick_params(a1.VARIANT_GAZEBO, a1.TICK_QP))
    seqs, speed = tick_inputs(B, 1, 2)
    tau, _ = tick.run(DT, *(seqs[k][0] for k in a1.TICK_INPUTS[:-1]), speed)
    assert np.isfinite(tau).all()
    e.close()                       # before the tick: the engine destroys the tick, then its handle
    assert tick.t is None and e.h is None
    tick.close()                    # and the tick's own close and finaliser do nothing more
    del tick
    e2 = a1.Engine(a1.default_config())   # the device is still usable
    e2.close()
