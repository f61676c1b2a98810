"""The work queue of the class kernels on the GPU: every CTA claims its first QPs when it starts (claim_qps), later QPs are drawn
one at a time, and a CTA that finds its class's counter exhausted leaves.  Mixes whose trot count lands exactly on, one below and
one above the trot slots that fit next to the four-stance CTAs (8 per SM on the SMs that the four-stance class, 4 QPs per SM,
leaves free), at the benchmark batch and at a large one: every QP gets a status, and the results equal those of the same batch
solved in another order (outputs permuted back) bit for bit -- which CTA or slot serves a QP does not change its arithmetic."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TROT, FOUR, ONE = 0b1001, 0b1111, 0b0001


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _mix(a1, B, n2, n4, seed):
    """n2 trot QPs, n4 four-stance QPs, the rest one-stance, in a shuffled order"""
    assert n2 + n4 <= B
    st = a1.gen_states(B, 2, seed)
    contact = np.full(B, ONE, dtype=np.uint32)
    contact[:n2] = TROT
    contact[n2:n2 + n4] = FOUR
    st["contact"] = np.random.default_rng(seed).permutation(contact)
    return st


def _solve(a1, eng, st):
    B = st["contact"].shape[0]
    d = a1.DeviceBatch(eng, B)
    d.upload(st)
    sentinel_f = np.full((12, B), np.nan)
    sentinel_s = np.full(B, -7, dtype=np.int32)
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, d.f_body, sentinel_f.ctypes.data, sentinel_f.nbytes))
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, d.status, sentinel_s.ctypes.data, sentinel_s.nbytes))
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, d.iters, sentinel_s.ctypes.data, sentinel_s.nbytes))
    eng.sync()
    eng.solve_ptrs(B, d.inp, d.out)
    eng.sync()
    f, status = d.download()
    iters = np.zeros(B, dtype=np.int32)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, iters.ctypes.data, d.iters, iters.nbytes))
    eng.sync()
    return f, status, iters


def _cases(sm):
    # B = 1024: n4 four-stance QPs take ceil(n4 / 4) SMs, the trot class fits 8 * (sm - ceil(n4 / 4)) slots beside them;
    # n4 = 32 puts that boundary at B - 32 exactly on an H100 (132 SMs)
    n4 = 32
    edge = 8 * (sm - (n4 + 3) // 4)
    B = max(1024, edge + n4 + 1)
    out = [(B, edge - 1, n4), (B, edge, n4), (B, edge + 1, n4 - 1)]
    # a large batch: every class kernel launches one CTA per SM, so the claims of the grid cover 8 * sm trot and 4 * sm
    # four-stance QPs; counts on, below and above several such claim rounds
    for d in (-1, 0, 1):
        out.append((16384, 8 * sm * 5 + d, 4 * sm * 3 - d))
    return out


def test_claim_boundaries_every_qp_answered_and_order_independent(built, gpu_engine):
    import a1mpc as a1
    sm = _sm_count()
    for i, (B, n2, n4) in enumerate(_cases(sm)):
        st = _mix(a1, B, n2, n4, 300 + i)
        f, status, iters = _solve(a1, gpu_engine, st)
        assert (status >= 0).all() and (status <= a1.STATUS_NO_CONTACT).all(), (B, n2, n4, np.bincount(status[status >= 0]))
        assert np.isfinite(f).all() and (iters >= 0).all()
        perm = np.random.default_rng(i).permutation(B)
        sp = {k: (v[..., perm] if v.ndim == 2 else v[perm]) for k, v in st.items()}
        fp, sp_status, ip = _solve(a1, gpu_engine, sp)
        inv = np.argsort(perm)
        assert np.array_equal(fp[:, inv], f), (B, n2, n4, np.abs(fp[:, inv] - f).max())
        assert np.array_equal(sp_status[inv], status) and np.array_equal(ip[inv], iters), (B, n2, n4)
