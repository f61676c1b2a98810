// emu_dense.cpp -- the kernels of a1mpc_solve_dense_batch and a1mpc_grf_qp_batch (classify_kernel, mark_unsupported_kernel,
// dense_solve_kernel<NS,N>, grf_qp_kernel<NS> of a1mpc_dense.cu) on the CPU block emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY,
// next to emu_driver.cpp: the UNCHANGED device code, launched the way dense_solve_launch and grf_qp_launch launch it (classify, then
// the heaviest class first; at N = 20 the three- and four-foot classes marked unsupported).  A grid cap per class lets a few blocks loop
// over a class's QPs as the device's CTAs do once a class has more QPs than CTAs.
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include <algorithm>
#include <atomic>
#include <functional>
#include <thread>
#include <vector>

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_dense.cu"   // kernels only (host launchers are compiled out under A1MPC_EMU)

using namespace a1mpc;

namespace {

DevParams make_params(const a1mpc_config* cfg) {   // a1mpc_create() in a1mpc_api.cu
  DevParams P;
  std::memset(&P, 0, sizeof(P));
  P.N = cfg->horizon;
  P.max_iter = cfg->max_iter > 0 ? cfg->max_iter : 40;
  P.dt = cfg->dt; P.mu = cfg->mu; P.fzmax = cfg->fz_max; P.mass = cfg->mass;
  P.mu_switch = cfg->tol > 0.0 ? cfg->tol : MU_SWITCH_DEFAULT;
  for (int i = 0; i < 9; ++i) P.inertia[i] = cfg->inertia[i];
  for (int i = 0; i < 13; ++i) P.q2[i] = 2.0 * cfg->q[i];
  for (int i = 0; i < 12; ++i) P.r2[i] = 2.0 * cfg->r[i];
  return P;
}

// one kernel over `nq` QPs on `grid` blocks (max_blocks > 0: at most that many, each looping over its share; 0: one block per QP),
// the blocks spread over nthreads host threads
template <typename F>
void run_grid(int nq, int max_blocks, int nthreads, int threads_per_block, size_t smem, int order_mode, F&& kernel) {
  if (nq == 0) return;
  const int grid = max_blocks > 0 ? std::min(nq, max_blocks) : nq;
  std::atomic<int> next{0};
  auto worker = [&]() {
    for (;;) {
      const int bx = next.fetch_add(1);
      if (bx >= grid) break;
      a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)grid, 1, 1}, threads_per_block, smem, order_mode, kernel);
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < std::min(std::max(1, nthreads), grid); ++t) th.emplace_back(worker);
  worker();
  for (auto& t : th) t.join();
}

void per_qp(int B, const std::function<void()>& kernel) {   // thread-per-QP kernels: 128-thread blocks
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx) a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0, kernel);
}

template <int NS, int N>
void run_dense(const DevParams& P, int B, const double* H, const double* g, const uint32_t* contact, const int* list, const int* count,
               double* u, int32_t* status, int order_mode, int max_blocks, int nthreads) {
  run_grid(count[NS], max_blocks, nthreads, 32 * Geo<NS, N>::TW, DenseGeo<NS, N>::smem_bytes(), order_mode,
           [&]() { dense_solve_kernel<NS, N>(P, H, g, contact, list + (size_t)(NS - 1) * B, count, u, status); });
}

template <int NS>
void run_grf(const DevParams& P, int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot,
             const uint32_t* contact, const int* list, const int* count, double* f_body, int32_t* status, int order_mode, int max_blocks) {
  run_grid(count[NS], max_blocks, 1, 32, DenseGeo<NS, 1>::smem_bytes() + 72 * 8, order_mode,
           [&]() { grf_qp_kernel<NS>(P, root_acc, rot_z, rot, foot, contact, list + (size_t)(NS - 1) * B, count, f_body, status); });
}

}  // namespace

extern "C" {

// a1mpc_solve_dense_batch (QP-major host arrays H [B,n,n], g [B,n], u [B,n]).  order_mode: lane order between collectives (0 ascending,
// 1 descending, 2 pseudo-random); max_blocks: grid cap per class (0 = one block per QP); nthreads: host threads over a class's blocks
int emu_dense_solve(const a1mpc_config* cfg, int B, const double* H, const double* g, const uint32_t* contact, double* u, int32_t* status,
                    int order_mode, int max_blocks, int nthreads) {
  if (cfg->horizon != 10 && cfg->horizon != 20) return -1;
  const DevParams P = make_params(cfg);
  const int n = 12 * cfg->horizon;
  std::vector<int> list((size_t)4 * B, 0);
  int count[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  per_qp(B, [&]() { classify_kernel(B, contact, list.data(), count, u, n, status); });
  if (cfg->horizon == 20) {
    per_qp(B, [&]() { mark_unsupported_kernel(list.data() + (size_t)3 * B, count, 4, u, n, status); });
    per_qp(B, [&]() { mark_unsupported_kernel(list.data() + (size_t)2 * B, count, 3, u, n, status); });
    run_dense<2, 20>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
    run_dense<1, 20>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
    return 0;
  }
  run_dense<4, 10>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
  run_dense<3, 10>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
  run_dense<2, 10>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
  run_dense<1, 10>(P, B, H, g, contact, list.data(), count, u, status, order_mode, max_blocks, nthreads);
  return 0;
}

// a1mpc_grf_qp_batch (QP-major host arrays), max_blocks as above
int emu_dense_grf_qp(int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot, const uint32_t* contact,
                     double* f_body, int32_t* status, int order_mode, int max_blocks) {
  const DevParams P = grf_params();
  std::vector<int> list((size_t)4 * B, 0);
  int count[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  per_qp(B, [&]() { classify_kernel(B, contact, list.data(), count, f_body, 12, status); });
  run_grf<4>(P, B, root_acc, rot_z, rot, foot, contact, list.data(), count, f_body, status, order_mode, max_blocks);
  run_grf<3>(P, B, root_acc, rot_z, rot, foot, contact, list.data(), count, f_body, status, order_mode, max_blocks);
  run_grf<2>(P, B, root_acc, rot_z, rot, foot, contact, list.data(), count, f_body, status, order_mode, max_blocks);
  run_grf<1>(P, B, root_acc, rot_z, rot, foot, contact, list.data(), count, f_body, status, order_mode, max_blocks);
  return 0;
}

}  // extern "C"
