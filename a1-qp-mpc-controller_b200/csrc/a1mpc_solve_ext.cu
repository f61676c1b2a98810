// a1mpc_solve_ext.cu -- the fused kernel for BASELINE config 4 (an extension beyond the reference, which has a constant
// contact pattern over the horizon and world-z friction pyramids): per-step contact schedules + per-foot terrain normals.
// It is the 4-foot wrench-space kernel with absent foot-steps pinned to zero (identity rows), forces solved in each
// foot's terrain frame.
#include "a1mpc_internal.h"
#include "a1mpc_sched.cuh"

namespace a1mpc {

template <int N>
static cudaError_t setup_n(int sm_count, ClassLaunch& c) {
  using G = Geo<4, N, 1>;
  // N = 10: 4 warps per CTA like the other wrench-space classes (rendezvous before every factorisation); N = 20: one
  constexpr int WPC = (N == 10) ? A1MPC_WPC34 : 1;
  c.wpc = WPC;
  c.smem = G::smem_bytes(WPC);
  cudaError_t e = cudaFuncSetAttribute(solve_kernel<4, N, WPC, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, solve_kernel<4, N, WPC, 1, true>, 32 * WPC * Geo<4, N, 1>::TW, c.smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  c.max_ctas = occ * sm_count;
  c.supported = true;
  return cudaSuccess;
}

cudaError_t ext_setup(int horizon, int sm_count, ClassLaunch& c) { return horizon == 10 ? setup_n<10>(sm_count, c) : setup_n<20>(sm_count, c); }

void ext_launch(int horizon, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out) {
  int grid = (B + c.wpc - 1) / c.wpc;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  if (horizon == 10) solve_kernel<4, 10, A1MPC_WPC34, 1, true><<<grid, 32 * A1MPC_WPC34 * Geo<4, 10, 1>::TW, c.smem, st>>>(P, rec, count, out);
  else solve_kernel<4, 20, 1, 1, true><<<grid, 32 * Geo<4, 20, 1>::TW, c.smem, st>>>(P, rec, count, out);
}

// warm start of the scheduled call (a1mpc_solve_batch_ext_warm), N = 10: the general kernel with K more ints per slot for the guess
cudaError_t ext_warm_setup(int sm_count, ClassLaunch& c) {
  constexpr int WPC = A1MPC_WPC34;
  c.wpc = WPC;
  c.smem = ext_warm_smem_bytes<10, WPC>();
  cudaError_t e = cudaFuncSetAttribute(solve_kernel_ext_warm<10, WPC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, solve_kernel_ext_warm<10, WPC>, 32 * WPC * Geo<4, 10, 1>::TW, c.smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  c.max_ctas = occ * sm_count;
  c.supported = true;
  return cudaSuccess;
}

void ext_warm_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out,
                     uint32_t* warm, int shift) {
  int grid = (B + c.wpc - 1) / c.wpc;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  solve_kernel_ext_warm<10, A1MPC_WPC34><<<grid, 32 * A1MPC_WPC34 * Geo<4, 10, 1>::TW, c.smem, st>>>(P, rec, count, out, warm, shift);
}

cudaError_t sched2_setup(int sm_count, ClassLaunch& c) {
  constexpr int WPC = 4;
  c.wpc = WPC;
  c.smem = SchedGeo<10>::smem_bytes(WPC);
  cudaError_t e = cudaFuncSetAttribute(solve_kernel_sched2<10, WPC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, solve_kernel_sched2<10, WPC>, 32 * WPC, c.smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  c.max_ctas = occ * sm_count;
  c.supported = true;
  return cudaSuccess;
}

void sched2_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out) {
  int grid = (B + c.wpc - 1) / c.wpc;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  solve_kernel_sched2<10, 4><<<grid, 32 * 4, c.smem, st>>>(P, rec, count, out);
}

cudaError_t sched2_warm_setup(int sm_count, ClassLaunch& c) {
  constexpr int WPC = 4;
  c.wpc = WPC;
  c.smem = SchedGeo<10>::smem_bytes(WPC);   // the guess lives in the slot's c.exist, which this class does not use
  cudaError_t e = cudaFuncSetAttribute(solve_kernel_sched2_warm<10, WPC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, solve_kernel_sched2_warm<10, WPC>, 32 * WPC, c.smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  c.max_ctas = occ * sm_count;
  c.supported = true;
  return cudaSuccess;
}

void sched2_warm_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out,
                        uint32_t* warm, int shift) {
  int grid = (B + c.wpc - 1) / c.wpc;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  solve_kernel_sched2_warm<10, 4><<<grid, 32 * 4, c.smem, st>>>(P, rec, count, out, warm, shift);
}

}  // namespace a1mpc
