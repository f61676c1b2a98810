// oracle/stance_terrain_oracle.cpp -- TEST INFRASTRUCTURE, not product code.
//
// compute_grf's 12-force QP branch (oracle_grf_qp_single of a1mpc_oracle.cpp) with each foot's friction pyramid posed in that foot's
// terrain frame: the check of a1mpc_stance_qp_batch_ext.  The QP in the world forces is oracle_grf_qp_single's, term for term; it is
// transformed as solve_one_ext transforms the MPC's, P' = T^T P T and q' = T^T q over T = blockdiag of the four terrain frames, and the
// pyramid and fz bounds then act on the local forces.  The exact long-double solve and its KKT certificate are those of
// oracle_solve_dense (a 1-step problem at mu 0.7, fz in [0, 180]: the feasible set oracle_grf_qp_single hands the same solver).  With
// e_z normals every added product is exact, so the result is oracle_grf_qp_single's bit for bit.  Built by
// `make -C oracle -f stance_terrain.mk` (the top-level Makefile runs it), linked against the unchanged liba1mpc_oracle.so.
#include <atomic>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../include/a1mpc.h"

extern "C" int oracle_solve_dense(const a1mpc_config* cfg, const double* H, const double* g, uint32_t contact, int mode, double* u, double* info8);

namespace {

// the rotation taking world z to the unit normal n (about the horizontal axis z x n), row-major: terrain_frame of a1mpc_oracle.cpp
void terrain_frame(const double* n_in, double* R) {
  double nx = n_in[0], ny = n_in[1], nz = n_in[2];
  const double inv = 1.0 / std::sqrt(nx * nx + ny * ny + nz * nz);
  nx *= inv; ny *= inv; nz *= inv;
  const double k = 1.0 / (1.0 + nz);
  R[0] = 1 - nx * nx * k; R[1] = -nx * ny * k;    R[2] = nx;
  R[3] = -nx * ny * k;    R[4] = 1 - ny * ny * k; R[5] = ny;
  R[6] = -nx;             R[7] = -ny;             R[8] = nz;
}

}  // namespace

extern "C" {

// root_acc[6], rot_z[9], rot[9] row-major, foot[12] leg-major, contact mask, normals12 per foot (world frame, any length > 0; NULL = e_z);
// mode must be 0 (exact).  f_body[12] out, info8 as oracle_grf_qp_single (iters, verified, kkt_stat, kkt_prim, kkt_dual, rounds).
// Returns -1 for another mode.
int oracle_grf_qp_single_ext(const double* root_acc, const double* rot_z, const double* rot, const double* foot, uint32_t contact,
                             const double* normals12, int mode, double* f_body, double* info8) {
  if (mode != 0) return -1;
  const double Qd[6] = {1.0, 1.0, 1.0, 400.0, 400.0, 100.0};
  const double Rw = 1e-3;
  // inertia_inv 6x12 (A1RobotControl.cpp:394-399), as oracle_grf_qp_single builds it
  double Minv[6][12];
  double RzT[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) RzT[3 * j + i] = rot_z[3 * i + j];
  for (int i = 0; i < 4; ++i) {
    const double* v = &foot[3 * i];
    const double S[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
    double M3[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double s = 0;
        for (int k = 0; k < 3; ++k) s += RzT[3 * r + k] * S[3 * k + c];
        M3[3 * r + c] = s;
      }
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) {
        Minv[a][3 * i + b] = (a == b) ? 1.0 : 0.0;
        Minv[3 + a][3 * i + b] = M3[3 * a + b];
      }
  }
  double P[144], q[12];
  for (int i = 0; i < 12; ++i) {
    for (int j = 0; j < 12; ++j) {
      double s = (i == j) ? Rw : 0.0;
      for (int k = 0; k < 6; ++k) s += Minv[k][i] * Qd[k] * Minv[k][j];
      P[12 * i + j] = s;
    }
    double s = 0;
    for (int k = 0; k < 6; ++k) s += Minv[k][i] * Qd[k] * root_acc[k];
    q[i] = -s;
  }
  // P' = T^T P T, q' = T^T q (solve_one_ext's order: P T first, then T^T (P T))
  double Rf[4][9];
  for (int i = 0; i < 4; ++i) {
    double nn[3] = {0, 0, 1};
    if (normals12)
      for (int a = 0; a < 3; ++a) nn[a] = normals12[3 * i + a];
    terrain_frame(nn, Rf[i]);
  }
  double PT[144], Pl[144], ql[12];
  for (int r = 0; r < 12; ++r)
    for (int kf = 0; kf < 4; ++kf)
      for (int c2 = 0; c2 < 3; ++c2) {
        double sacc = 0;
        for (int a = 0; a < 3; ++a) sacc += P[12 * r + 3 * kf + a] * Rf[kf][3 * a + c2];
        PT[12 * r + 3 * kf + c2] = sacc;
      }
  for (int kf = 0; kf < 4; ++kf)
    for (int c2 = 0; c2 < 3; ++c2) {
      for (int col = 0; col < 12; ++col) {
        double sacc = 0;
        for (int a = 0; a < 3; ++a) sacc += Rf[kf][3 * a + c2] * PT[12 * (3 * kf + a) + col];
        Pl[12 * (3 * kf + c2) + col] = sacc;
      }
      double sq = 0;
      for (int a = 0; a < 3; ++a) sq += Rf[kf][3 * a + c2] * q[3 * kf + a];
      ql[3 * kf + c2] = sq;
    }
  a1mpc_config cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.horizon = 1; cfg.precision = 64; cfg.mu = 0.7; cfg.fz_min = 0.0; cfg.fz_max = 180.0;   // A1RobotControl.cpp:13-15
  for (int k = 0; k < 13; ++k) cfg.q[k] = 1.0;   // unused by the solve of a given P, q
  for (int k = 0; k < 12; ++k) cfg.r[k] = 1.0;
  double sol[12] = {0}, info[8];
  oracle_solve_dense(&cfg, Pl, ql, contact, 0, sol, info);
  if (info8) std::memcpy(info8, info, sizeof(info));
  // local -> world -> body (:439-444)
  for (int i = 0; i < 4; ++i) {
    const double* R = Rf[i];
    double uw[3];
    for (int a = 0; a < 3; ++a) uw[a] = R[3 * a] * sol[3 * i] + R[3 * a + 1] * sol[3 * i + 1] + R[3 * a + 2] * sol[3 * i + 2];
    for (int a = 0; a < 3; ++a) f_body[3 * i + a] = rot[0 * 3 + a] * uw[0] + rot[1 * 3 + a] * uw[1] + rot[2 * 3 + a] * uw[2];
  }
  return 0;
}

// oracle_grf_qp_single_ext for a batch on host threads, batch-major like a1mpc_stance_qp_batch_ext (ld = B): root_acc [6][B], rot_z [9][B],
// rot [9][B], foot [12][B], contact [B], normals [12][B]; out f_body [12][B], info [B][8].  A robot without a stance foot gets zero forces
// and info[1] = 1 without a solve.
int oracle_grf_qp_batch_ext(int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot, const uint32_t* contact,
                            const double* normals, int nthreads, double* f_body, double* info) {
  if (nthreads < 1) nthreads = 1;
  std::atomic<int> next(0);
  auto work = [&]() {
    for (;;) {
      const int b = next.fetch_add(1);
      if (b >= B) break;
      const size_t ld = (size_t)B;
      double acc[6], rz[9], R[9], ft[12], nn[12], f[12] = {0}, in8[8] = {0};
      for (int k = 0; k < 6; ++k) acc[k] = root_acc[k * ld + b];
      for (int k = 0; k < 9; ++k) { rz[k] = rot_z[k * ld + b]; R[k] = rot[k * ld + b]; }
      for (int k = 0; k < 12; ++k) { ft[k] = foot[k * ld + b]; nn[k] = normals[k * ld + b]; }
      if (contact[b] & 15u) oracle_grf_qp_single_ext(acc, rz, R, ft, contact[b] & 15u, nn, 0, f, in8);
      else in8[1] = 1.0;
      for (int k = 0; k < 12; ++k) f_body[k * ld + b] = f[k];
      std::memcpy(info + (size_t)b * 8, in8, sizeof(in8));
    }
  };
  if (nthreads == 1) { work(); return 0; }
  std::vector<std::thread> th;
  for (int t = 0; t < nthreads; ++t) th.emplace_back(work);
  for (auto& t : th) t.join();
  return 0;
}

}  // extern "C"
