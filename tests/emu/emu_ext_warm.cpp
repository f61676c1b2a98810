// emu_ext_warm.cpp -- the warm-started kernels of a1mpc_solve_batch_ext_warm on the CPU block emulator of cuda_emu.h.
// TEST INFRASTRUCTURE ONLY, next to emu_driver.cpp (which runs the cold kernels and the constant-pattern warm start): the
// UNCHANGED device code, launched the way a1mpc_api.cu launches it (warm_forget_no_contact_kernel, pack kernel, solve kernel).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include <atomic>
#include <thread>

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_misc.cuh"
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_sched.cuh"

using namespace a1mpc;

namespace {

DevParams make_params(const a1mpc_config* cfg) {   // a1mpc_create() in a1mpc_api.cu
  DevParams P;
  P.N = cfg->horizon;
  P.max_iter = cfg->max_iter > 0 ? cfg->max_iter : 40;
  P.dt = cfg->dt; P.mu = cfg->mu; P.fzmax = cfg->fz_max; P.mass = cfg->mass;
  P.mu_switch = cfg->tol > 0.0 ? cfg->tol : MU_SWITCH_DEFAULT;
  for (int i = 0; i < 9; ++i) P.inertia[i] = cfg->inertia[i];
  for (int i = 0; i < 13; ++i) P.q2[i] = 2.0 * cfg->q[i];
  for (int i = 0; i < 12; ++i) P.r2[i] = 2.0 * cfg->r[i];
  return P;
}

// thread-per-robot prologue of the call: clear the slots of robots without contact, pack the extended records (queue 5)
void prologue(const DevInputs& din, const uint32_t* sched, const double* normals, int B, uint32_t* warm, std::vector<double>& rec, int* count,
              const DevOutputs& dout, int horizon) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx) {
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0,
                     [&]() { warm_forget_no_contact_kernel(din, sched, B, warm, horizon); });
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0,
                     [&]() { pack_ext_kernel(din, sched, normals, B, rec.data(), count, dout, horizon); });
  }
}

// persistent grid of ~2 QPs per warp (exercises the persistent loop and the CTA rendezvous), blocks spread over host threads
template <class F>
void run_grid(int nq, int wpc, int threads, size_t smem, int order_mode, int nthreads, F kernel) {
  if (nq == 0) return;
  const int grid = std::max(1, (nq + 2 * wpc - 1) / (2 * wpc));
  std::atomic<int> next{0};
  auto worker = [&]() {
    for (;;) {
      const int bx = next.fetch_add(1);
      if (bx >= grid) break;
      a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)grid, 1, 1}, threads, smem, order_mode, kernel);
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < std::max(1, nthreads); ++t) th.emplace_back(worker);
  worker();
  for (auto& t : th) t.join();
}

}  // namespace

extern "C" {

// a1mpc_solve_batch_ext_warm on the general four-leg kernel (solve_kernel_ext_warm<10, A1MPC_WPC34>), host pointers; N = 10.
// warm: B * (4 + 4 N) u32, the library's layout.  order_mode: lane order between collectives (0 ascending, 1 descending, 2 random)
int emu_solve_ext_warm(const a1mpc_config* cfg, int B, const a1mpc_inputs* in, const uint32_t* sched, const double* normals,
                       const a1mpc_outputs* o, int order_mode, int nthreads, uint32_t* warm, int shift) {
  if (cfg->horizon != 10 || !warm || (!sched && !normals)) return -1;
  constexpr int N = 10, WPC = A1MPC_WPC34;
  const DevParams P = make_params(cfg);
  const DevInputs din{in->x0, in->rot, in->foot, in->ref, in->contact, in->ld};
  const DevOutputs dout{o->f_body, o->status, o->iters, o->u_full, o->ld};
  int count[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // [0..7] class counts, [8..15] queue counters (next_qp)
  std::vector<double> rec((size_t)B * REC_EXT_DOUBLES + 2);
  prologue(din, sched, normals, B, warm, rec, count, dout, N);
  run_grid(count[5], WPC, 32 * WPC * Geo<4, N, 1>::TW, ext_warm_smem_bytes<N, WPC>(), order_mode, nthreads,
           [&]() { solve_kernel_ext_warm<N, WPC>(P, rec.data(), count, dout, warm, shift); });
  return 0;
}

// the same on the compacted two-feet kernel (solve_kernel_sched2_warm<10, 4>); every robot must have exactly two stance feet in
// every step
int emu_solve_sched2_warm(const a1mpc_config* cfg, int B, const a1mpc_inputs* in, const uint32_t* sched, const double* normals,
                          const a1mpc_outputs* o, int order_mode, int nthreads, uint32_t* warm, int shift) {
  if (cfg->horizon != 10 || !sched || !warm) return -1;
  for (int st = 0; st < 10; ++st)
    for (int b = 0; b < B; ++b)
      if (__builtin_popcount(sched[(size_t)st * in->ld + b] & 15u) != 2) return -2;
  constexpr int N = 10, WPC = 4;
  const DevParams P = make_params(cfg);
  const DevInputs din{in->x0, in->rot, in->foot, in->ref, in->contact, in->ld};
  const DevOutputs dout{o->f_body, o->status, o->iters, o->u_full, o->ld};
  int count[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  std::vector<double> rec((size_t)B * REC_EXT_DOUBLES + 2);
  prologue(din, sched, normals, B, warm, rec, count, dout, N);
  count[6] = count[5];
  run_grid(count[6], WPC, 32 * WPC, SchedGeo<N>::smem_bytes(WPC), order_mode, nthreads,
           [&]() { solve_kernel_sched2_warm<N, WPC>(P, rec.data(), count, dout, warm, shift); });
  return 0;
}

}  // extern "C"
