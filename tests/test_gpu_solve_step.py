"""The solve step (a1mpc_api.cu, enqueue_solve: pack_kernel, then the four class kernels on their own streams) across the class mixes
and call sequences a controller produces: batches of one class, of every class and of none; class counts around a whole number of
CTAs and beyond the CTAs resident on the device; a batch that outgrows the handle's records; cold and warm calls alternating;
input and output arrays that change on every call with no synchronisation between calls; host-pointer calls; a horizon-20 handle;
profiling on and off.  Every case checks status and forces against the oracle, and that the same batch solved in a permuted order
gives the same outputs (permuted back) bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL_F = 1e-4
ONE, TROT, THREE, FOUR = 0b0001, 0b1001, 0b0111, 0b1111
WPC = {ONE: 8, TROT: 8, THREE: 4, FOUR: 4}   # QPs per CTA of the N = 10 class kernels (A1MPC_WPC1 / 2 / 34)


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def O(built):
    from oracle import oracle_py
    return oracle_py


def _states(a1, counts, seed, config_id=2):
    """a batch with counts[pattern] QPs of each contact pattern, shuffled"""
    B = sum(counts.values())
    st = a1.gen_states(B, config_id, seed)
    st["contact"] = np.random.default_rng(seed).permutation(np.concatenate([np.full(n, p, dtype=np.uint32) for p, n in counts.items()]))
    return st


def _permuted(st, perm):
    return {k: (v[..., perm] if v.ndim == 2 else v[perm]) for k, v in st.items()}


def _device_solve(a1, eng, st):
    B = st["contact"].shape[0]
    d = a1.DeviceBatch(eng, B)
    d.upload(st)
    eng.solve_ptrs(B, d.inp, d.out)
    f, status = d.download()
    d.free()
    return f, status


def _check_oracle(a1, O, st, f, status, horizon=10):
    from common import obatch
    fo, info = O.compute_grf_batch(O.make_config(horizon=horizon), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    nc = (st["contact"] & 15) == 0
    assert (status[nc] == a1.STATUS_NO_CONTACT).all() and (f[:, nc] == 0).all()
    assert (status[~nc] == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= TOL_F


def _check(a1, O, eng, st, seed, horizon=10):
    """solve on device pointers, check against the oracle, solve permuted: bit-identical; returns the outputs"""
    f, status = _device_solve(a1, eng, st)
    _check_oracle(a1, O, st, f, status, horizon)
    perm = np.random.default_rng(seed).permutation(st["contact"].shape[0])
    fp, sp = _device_solve(a1, eng, _permuted(st, perm))
    inv = np.argsort(perm)
    assert np.array_equal(fp[:, inv], f) and np.array_equal(sp[inv], status)
    return f, status


@pytest.mark.parametrize("pattern", [ONE, TROT, THREE, FOUR])
def test_one_class_only(a1, O, gpu_engine, pattern):
    n0 = gpu_engine.launches()
    _check(a1, O, gpu_engine, _states(a1, {pattern: 200}, 11 + pattern), 1)
    assert gpu_engine.launches() - n0 == 2 * 5   # two solves: pack and the four class kernels each


def test_all_four_classes(a1, O, gpu_engine):
    _check(a1, O, gpu_engine, _states(a1, {ONE: 40, TROT: 600, THREE: 50, FOUR: 100}, 21), 2)


def test_no_contact_batch_then_a_full_batch(a1, O, gpu_engine):
    st = _states(a1, {0: 300}, 31)
    f, status = _check(a1, O, gpu_engine, st, 3)
    assert (status == a1.STATUS_NO_CONTACT).all()
    _check(a1, O, gpu_engine, _states(a1, {ONE: 9, TROT: 100, THREE: 9, FOUR: 20, 0: 5}, 32), 4)


@pytest.mark.parametrize("d", [-1, 0, 1])
def test_class_counts_around_a_whole_number_of_ctas(a1, O, gpu_engine, d):
    """every class count at WPC * k + d: the last CTA of each class is full, one short or holds one QP"""
    counts = {p: WPC[p] * k + d for p, k in ((ONE, 2), (TROT, 5), (THREE, 3), (FOUR, 7))}
    _check(a1, O, gpu_engine, _states(a1, counts, 40 + d), 5 + d)


def test_class_larger_than_the_resident_ctas(a1, O, gpu_engine):
    """more trot and four-stance QPs than max_ctas * WPC slots (one CTA per SM): the slots draw the rest from the queue"""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    _check(a1, O, gpu_engine, _states(a1, {TROT: 8 * sm + 300, FOUR: 4 * sm + 50}, 51), 9)


def test_batch_growing_on_one_handle_reallocates_the_records(a1, O):
    """B past the record capacity (1024, 2048) reallocates the records of the handle"""
    eng = a1.Engine(a1.default_config())
    for i, B in enumerate((64, 1100, 2100)):
        st = a1.gen_states(B, 4, 60 + i)
        _check(a1, O, eng, st, 60 + i)
        f, status, _ = eng.solve(st)   # host pointers on the same handle
        g, s = _device_solve(a1, eng, st)
        assert np.array_equal(f, g) and np.array_equal(status, s)
    eng.close()


def test_cold_and_warm_alternating_on_one_handle(a1, O):
    """cold and warm calls on one handle share its records and counters; alternating them keeps both right"""
    from common import obatch
    eng = a1.Engine(a1.default_config())
    B = 512
    warm = eng.warm_alloc(B)
    st = _states(a1, {ONE: 20, TROT: 400, THREE: 30, FOUR: 62}, 71)
    fo, info = O.compute_grf_batch(O.make_config(), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    cold, warm_out = None, []
    for i in range(3):
        f, status, _ = eng.solve(st)
        assert (status == a1.STATUS_OPTIMAL).all() and np.abs(f - fo).max() <= TOL_F
        if cold is None:
            cold = f
        assert np.array_equal(f, cold)
        fw, sw, _ = eng.solve_warm(st, warm, shift=0)
        assert (sw == a1.STATUS_OPTIMAL).all() and np.abs(fw - fo).max() <= TOL_F
        warm_out.append((fw, sw))
    # the warm path permuted: a guess belongs to its robot, so the same two calls on the permuted batch give the same outputs
    perm = np.random.default_rng(7).permutation(B)
    warm2 = eng.warm_alloc(B)
    sp = _permuted(st, perm)
    inv = np.argsort(perm)
    for k in range(2):
        fw2, sw2, _ = eng.solve_warm(sp, warm2, shift=0)
        assert np.array_equal(fw2[:, inv], warm_out[k][0]) and np.array_equal(sw2[inv], warm_out[k][1])
    for w in (warm, warm2):
        a1._check(a1.lib().a1mpc_device_free(eng.h, w))
    eng.close()


def test_pointers_change_every_call_without_sync(a1, O, gpu_engine):
    """four device batches solved round robin, twice, with no synchronisation between the calls"""
    batches = [_states(a1, {ONE: 10 + r, TROT: 200 + 30 * r, THREE: 5 + r, FOUR: 40 - 3 * r, 0: r}, 80 + r) for r in range(4)]
    refs = [_device_solve(a1, gpu_engine, st) for st in batches]
    dev = []
    for st in batches:
        d = a1.DeviceBatch(gpu_engine, st["contact"].shape[0])
        d.upload(st)
        dev.append(d)
    for _ in range(2):
        for d in dev:
            gpu_engine.solve_ptrs(d.B, d.inp, d.out)
    gpu_engine.sync()
    for st, d, (f, status) in zip(batches, dev, refs):
        g, s = d.download()
        assert np.array_equal(g, f) and np.array_equal(s, status)
        _check_oracle(a1, O, st, g, s)
        d.free()


def test_host_pointer_calls(a1, O, gpu_engine):
    st = _states(a1, {ONE: 17, TROT: 301, THREE: 13, FOUR: 45, 0: 3}, 91)
    f, status, _ = gpu_engine.solve(st)
    _check_oracle(a1, O, st, f, status)
    perm = np.random.default_rng(91).permutation(st["contact"].shape[0])
    fp, sp, _ = gpu_engine.solve(_permuted(st, perm))
    inv = np.argsort(perm)
    assert np.array_equal(fp[:, inv], f) and np.array_equal(sp[inv], status)
    g, s = _device_solve(a1, gpu_engine, st)
    assert np.array_equal(g, f) and np.array_equal(s, status)


def test_horizon_20_handle(a1, O):
    eng = a1.Engine(a1.default_config(horizon=20))
    _check(a1, O, eng, _states(a1, {ONE: 7, TROT: 60, THREE: 9, FOUR: 20, 0: 2}, 101), 11, horizon=20)
    _check(a1, O, eng, _states(a1, {TROT: 50}, 102), 12, horizon=20)
    eng.close()


def test_profiling_on_and_off_gives_identical_outputs(a1, O, gpu_engine):
    """profiling records timing events around the class kernels and changes nothing they compute"""
    st = _states(a1, {TROT: 500, FOUR: 60}, 111)
    f, status = _device_solve(a1, gpu_engine, st)
    gpu_engine.profile_begin(3)
    outs = [_device_solve(a1, gpu_engine, st) for _ in range(3)]
    ms, n = gpu_engine.profile_end()
    assert n == 3 and np.isfinite(ms).all() and (ms >= 0).all()
    assert ms[1] > 0 and ms[3] > 0, ms      # the trot and four-stance kernels ran between their events
    for g, s in outs:
        assert np.array_equal(g, f) and np.array_equal(s, status)
    g, s = _device_solve(a1, gpu_engine, st)
    assert np.array_equal(g, f) and np.array_equal(s, status)
    _check_oracle(a1, O, st, f, status)
