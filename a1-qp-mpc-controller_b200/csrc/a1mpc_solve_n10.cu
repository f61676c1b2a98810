// a1mpc_solve_n10.cu -- instantiations of the fused kernel for PLAN_HORIZON = 10 (A1Params.h:26)
#include "a1mpc_internal.h"

namespace a1mpc {

template <int NS, int N, int WPC, int LSM>
static cudaError_t setup_one(int sm_count, ClassLaunch& c) {
  using G = Geo<NS, N, LSM>;
  c.wpc = WPC;
  c.smem = G::smem_bytes(WPC);
  cudaError_t e = cudaFuncSetAttribute(solve_kernel<NS, N, WPC, LSM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, solve_kernel<NS, N, WPC, LSM>, 32 * WPC * G::TW, c.smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorLaunchOutOfResources;
  c.max_ctas = occ * sm_count;
  c.supported = true;
  return cudaSuccess;
}

template <int NS, int N, int WPC, int LSM>
static cudaError_t setup_one_warm(const ClassLaunch& c) {
  return cudaFuncSetAttribute(solve_kernel_warm<NS, N, WPC, LSM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem);
}

template <int NS, int N, int WPC, int LSM>
static void launch_one_warm(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count,
                            const DevOutputs& out, uint32_t* warm, int shift) {
  int grid = (B + WPC - 1) / WPC;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  solve_kernel_warm<NS, N, WPC, LSM><<<grid, 32 * WPC * Geo<NS, N, LSM>::TW, c.smem, st>>>(P, rec, count, out, warm, shift);
}

template <int NS, int N, int WPC, int LSM>
static void launch_one(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out) {
  int grid = (B + WPC - 1) / WPC;
  if (grid > c.max_ctas) grid = c.max_ctas;
  if (grid < 1) grid = 1;
  solve_kernel<NS, N, WPC, LSM><<<grid, 32 * WPC * Geo<NS, N, LSM>::TW, c.smem, st>>>(P, rec, count, out);
}

#ifndef A1MPC_HORIZON
#define A1MPC_HORIZON 10
#endif

#if A1MPC_HORIZON == 10
cudaError_t fused_setup_n10(int sm_count, ClassLaunch (&cls)[5]) {
  cudaError_t e;
  if ((e = setup_one<1, 10, A1MPC_WPC1, 0>(sm_count, cls[1])) != cudaSuccess) return e;
  if ((e = setup_one<2, 10, A1MPC_WPC2, 0>(sm_count, cls[2])) != cudaSuccess) return e;
  if ((e = setup_one<3, 10, A1MPC_WPC34, 1>(sm_count, cls[3])) != cudaSuccess) return e;
  if ((e = setup_one<4, 10, A1MPC_WPC34, 1>(sm_count, cls[4])) != cudaSuccess) return e;
  if ((e = setup_one_warm<1, 10, A1MPC_WPC1, 0>(cls[1])) != cudaSuccess) return e;
  if ((e = setup_one_warm<2, 10, A1MPC_WPC2, 0>(cls[2])) != cudaSuccess) return e;
  if ((e = setup_one_warm<3, 10, A1MPC_WPC34, 1>(cls[3])) != cudaSuccess) return e;
  if ((e = setup_one_warm<4, 10, A1MPC_WPC34, 1>(cls[4])) != cudaSuccess) return e;
  return cudaSuccess;
}
void fused_launch_n10_warm(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count,
                           const DevOutputs& out, uint32_t* warm, int shift) {
  if (ns == 1) launch_one_warm<1, 10, A1MPC_WPC1, 0>(c, st, B, P, rec, count, out, warm, shift);
  if (ns == 2) launch_one_warm<2, 10, A1MPC_WPC2, 0>(c, st, B, P, rec, count, out, warm, shift);
  if (ns == 3) launch_one_warm<3, 10, A1MPC_WPC34, 1>(c, st, B, P, rec, count, out, warm, shift);
  if (ns == 4) launch_one_warm<4, 10, A1MPC_WPC34, 1>(c, st, B, P, rec, count, out, warm, shift);
}
void fused_launch_n10(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out) {
  if (ns == 1) launch_one<1, 10, A1MPC_WPC1, 0>(c, st, B, P, rec, count, out);
  if (ns == 2) launch_one<2, 10, A1MPC_WPC2, 0>(c, st, B, P, rec, count, out);
  if (ns == 3) launch_one<3, 10, A1MPC_WPC34, 1>(c, st, B, P, rec, count, out);
  if (ns == 4) launch_one<4, 10, A1MPC_WPC34, 1>(c, st, B, P, rec, count, out);
}
#else
// warps per CTA of the N = 20 classes: 69.8 KB (NS = 2) / 117.8 KB (NS = 4, wrench) of shared memory per warp allow 3 / 1 per SM
#ifndef A1MPC_N20_WPC1
#define A1MPC_N20_WPC1 2
#endif
#ifndef A1MPC_N20_WPC2
#define A1MPC_N20_WPC2 3   // one CTA of three warps with the rendezvous instead of three independent one-warp CTAs:
#endif                     // one instruction-cache fill serves the three warps
#ifndef A1MPC_N20_WPC34
#define A1MPC_N20_WPC34 2  // wrench classes at N = 20: 106.5 KB per warp since B_k is no longer stored -> two warps per SM instead of one
#endif
cudaError_t fused_setup_n20(int sm_count, ClassLaunch (&cls)[5]) {
  cudaError_t e;
  if ((e = setup_one<1, 20, A1MPC_N20_WPC1, 0>(sm_count, cls[1])) != cudaSuccess) return e;
  if ((e = setup_one<2, 20, A1MPC_N20_WPC2, 0>(sm_count, cls[2])) != cudaSuccess) return e;
  if ((e = setup_one<3, 20, A1MPC_N20_WPC34, 1>(sm_count, cls[3])) != cudaSuccess) return e;
  if ((e = setup_one<4, 20, A1MPC_N20_WPC34, 1>(sm_count, cls[4])) != cudaSuccess) return e;
  return cudaSuccess;
}
void fused_launch_n20(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out) {
  if (ns == 1) launch_one<1, 20, A1MPC_N20_WPC1, 0>(c, st, B, P, rec, count, out);
  if (ns == 2) launch_one<2, 20, A1MPC_N20_WPC2, 0>(c, st, B, P, rec, count, out);
  if (ns == 3) launch_one<3, 20, A1MPC_N20_WPC34, 1>(c, st, B, P, rec, count, out);
  if (ns == 4) launch_one<4, 20, A1MPC_N20_WPC34, 1>(c, st, B, P, rec, count, out);
}
#endif

}  // namespace a1mpc
