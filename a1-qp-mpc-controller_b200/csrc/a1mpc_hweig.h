// a1mpc_hweig.h -- simultaneous diagonalisation of the condensed double integrator's tables (plain C++, fp64, constexpr).
//   T0[a][b] = N - max(a,b)                          (positive definite)
//   T1[a][b] = sum_{i>=max(a,b)} (i-a)(i-b)          (a Gram matrix: positive semidefinite, singular)
// hw_eig<N>() returns U and lambda with U' T0 U = I and U' T1 U = diag(lambda), lambda >= 0, so that the wrench-space Hessian
// Hw = T0 (x) Q0 + T1 (x) Q1' has the inverse (U (x) I6) blockdiag_s (Q0 + lambda_s Q1')^-1 (U' (x) I6).
// T0 = P P' with P[a][i] = [a <= i], and P^-1 = I - J (J the shift above the diagonal), so
//   C = P^-1 T1 P^-T = [N - 1 - max(a,b)]   (exact integers),   C = W diag(lambda) W'   (cyclic Jacobi),   U = P^-T W.
// The tables depend on N alone: they are evaluated by the compiler and stored into the kernels as constants.
#pragma once

#if defined(__CUDACC__)
#define A1MPC_HD __host__ __device__
#else
#define A1MPC_HD
#endif

namespace a1mpc {

template <int N>
struct HwEig {
  double v[N * N + N];   // U row-major (U[a][s] at a * N + s), then lambda_s at N * N + s
};

A1MPC_HD constexpr double cx_abs(double x) { return x < 0.0 ? -x : x; }
// Newton's iteration from above: decreases monotonically until it reaches the rounded root
A1MPC_HD constexpr double cx_sqrt(double x) {
  if (!(x > 0.0)) return 0.0;
  double y = x > 1.0 ? x : 1.0;
  for (int i = 0; i < 2000; ++i) {
    const double yn = 0.5 * (y + x / y);
    if (!(yn < y)) break;
    y = yn;
  }
  return y;
}

template <int N>
A1MPC_HD constexpr HwEig<N> hw_eig() {
  double a[N][N] = {}, w[N][N] = {};
  double fro = 0.0;
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) {
      a[i][j] = (double)(N - 1 - (i > j ? i : j));
      w[i][j] = (i == j) ? 1.0 : 0.0;
      fro += a[i][j] * a[i][j];
    }
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < N; ++p)
      for (int q = p + 1; q < N; ++q) off += a[p][q] * a[p][q];
    if (off <= 1e-34 * fro) break;
    for (int p = 0; p < N; ++p)
      for (int q = p + 1; q < N; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (cx_abs(theta) + cx_sqrt(theta * theta + 1.0));
        const double c = 1.0 / cx_sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < N; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        a[p][q] = 0.0;
        a[q][p] = 0.0;
        for (int k = 0; k < N; ++k) {
          const double wkp = w[k][p], wkq = w[k][q];
          w[k][p] = c * wkp - s * wkq;
          w[k][q] = s * wkp + c * wkq;
        }
      }
  }
  HwEig<N> r{};
  for (int i = 0; i < N; ++i)
    for (int s = 0; s < N; ++s) r.v[i * N + s] = w[i][s] - (i > 0 ? w[i - 1][s] : 0.0);
  for (int s = 0; s < N; ++s) r.v[N * N + s] = a[s][s] > 0.0 ? a[s][s] : 0.0;   // C is PSD: a rounding below zero is zero
  return r;
}

}  // namespace a1mpc
