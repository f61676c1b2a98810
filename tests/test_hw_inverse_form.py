"""The Hw^-1 + S form of the wrench-space solve (WrenchLS, HWI) and its fall-back.

The form needs U' T0 U = I, U' T1 U = diag(lambda) (a1mpc_hweig.h, evaluated at compile time) and Q0 = diag(2 q[6..11]) > 0;
a handle with a zero in q[6..11] keeps the Ls form.  Both are checked against the oracle, on the emulator and on the GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
from common import obatch  # noqa: E402

CHECK_SRC = r"""
#include <cmath>
#include <cstdio>
#include "a1mpc_hweig.h"
template <int N> void check() {
  constexpr a1mpc::HwEig<N> t = a1mpc::hw_eig<N>();
  double e0 = 0, e1 = 0, t1max = 0, lmin = 1e300;
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      double s0 = 0, s1 = 0;
      for (int a = 0; a < N; ++a)
        for (int b = 0; b < N; ++b) {
          const int m = a > b ? a : b;
          double t1 = 0;
          for (int k = m; k < N; ++k) t1 += (k - a) * (k - b);
          t1max = std::fmax(t1max, t1);
          s0 += t.v[a * N + i] * (N - m) * t.v[b * N + j];
          s1 += t.v[a * N + i] * t1 * t.v[b * N + j];
        }
      e0 = std::fmax(e0, std::fabs(s0 - (i == j)));
      e1 = std::fmax(e1, std::fabs(s1 - (i == j ? t.v[N * N + i] : 0.0)));
    }
  for (int s = 0; s < N; ++s) lmin = std::fmin(lmin, t.v[N * N + s]);
  std::printf("%d %.3e %.3e %.3e\n", N, e0, e1 / t1max, lmin);
}
int main() { check<10>(); check<20>(); }
"""


def test_hw_tables_diagonalise_t0_and_t1(tmp_path):
    src = tmp_path / "hw_check.cpp"
    src.write_text(CHECK_SRC)
    exe = tmp_path / "hw_check"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "a1-qp-mpc-controller_b200", "csrc"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    for line in filter(None, out):
        n, e0, e1, lmin = line.split()
        assert float(e0) <= 1e-14, line            # U' T0 U = I
        assert float(e1) <= 1e-14, line            # U' T1 U = diag(lambda), relative to max |T1|
        assert float(lmin) >= 0.0, line


def _zero_q(a1, horizon):
    q = list(a1.default_config(horizon=horizon).q)
    q[6] = 0.0   # no weight on the roll rate: Q0 is singular, so is Q0 + 0 * Q1'
    return q


def _states(a1, B, stream):
    st = a1.gen_states(B, 2, stream)
    pats = np.array([15, 7, 11, 13, 14], dtype=np.uint32)   # the wrench-space classes
    st["contact"] = pats[np.arange(B) % len(pats)]
    return st


@pytest.mark.parametrize("horizon,B", [(10, 40), (20, 10)])
def test_zero_velocity_weight_on_emulator(horizon, B):
    import emu_py as E
    from oracle import oracle_py as O
    a1 = E.a1mpc
    q = _zero_q(a1, horizon)
    st = _states(a1, B, 91)
    f, status, iters, stats = E.solve(a1.default_config(horizon=horizon, q=q), st, order=2)
    fo, info = O.compute_grf_batch(O.make_config(horizon=horizon, q=tuple(q)), obatch(O, st), O.MODE_EXACT, nthreads=4)
    assert (status == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= 1e-7


@pytest.mark.gpu
@pytest.mark.parametrize("horizon,B", [(10, 1024), (20, 256)])
@pytest.mark.parametrize("zero_q", [False, True])
def test_wrench_forms_on_gpu(built, horizon, B, zero_q):
    import a1mpc as a1
    from oracle import oracle_py as O
    q = _zero_q(a1, horizon) if zero_q else list(a1.default_config(horizon=horizon).q)
    st = _states(a1, B, 93)
    eng = a1.Engine(a1.default_config(horizon=horizon, q=q))
    f, status, iters = eng.solve(st)
    eng.close()
    fo, info = O.compute_grf_batch(O.make_config(horizon=horizon, q=tuple(q)), obatch(O, st), O.MODE_EXACT, nthreads=O.hardware_threads())
    assert (status == a1.STATUS_OPTIMAL).all(), np.bincount(status)
    assert np.abs(f - fo).max() <= 1e-7
