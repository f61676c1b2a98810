// emu_stance_terrain.cpp -- the kernels of a1mpc_stance_qp_batch_ext (stance_pack_kernel, stance_qp_ext_kernel<NS> of a1mpc_dense.cu) and
// of a1mpc_surface_normals_batch (surface_normals_kernel of a1mpc_swing.cuh) on the CPU block emulator of cuda_emu.h.  TEST
// INFRASTRUCTURE ONLY, next to emu_stance.cpp: the UNCHANGED device code, launched the way stance_qp_launch and a1mpc_api.cu launch it
// (pack and normals: 128-thread blocks; then one warp per QP, heaviest class first).  Host arrays, leading dimension ld.
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include <vector>

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_dense.cu"   // kernels only (host launchers are compiled out under A1MPC_EMU)
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_swing.cuh"

using namespace a1mpc;

namespace {
template <int NS>
void run_stance(const DevParams& P, int B, const double* rec, const uint32_t* contact, const int* list, const int* count, const double* normals,
                double* f_body, size_t ld, int32_t* status, int order_mode) {
  const int nq = count[NS];
  for (int bx = 0; bx < nq; ++bx) {
    if (normals)
      a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)nq, 1, 1}, 32, DenseGeo<NS, 1>::smem_bytes() + 84 * 8, order_mode,
                       [&]() { stance_qp_ext_kernel<NS>(P, rec, contact, list + (size_t)(NS - 1) * B, count, normals, f_body, ld, status); });
    else
      a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)nq, 1, 1}, 32, DenseGeo<NS, 1>::smem_bytes() + 72 * 8, order_mode,
                       [&]() { stance_qp_kernel<NS>(P, rec, contact, list + (size_t)(NS - 1) * B, count, f_body, ld, status); });
  }
}
}  // namespace

extern "C" {

// a1mpc_stance_qp_batch_ext (host arrays): normals [12][ld], or NULL for a1mpc_stance_qp_batch; gains9 = kd_linear, kp_angular,
// kd_angular; root_acc may be NULL
int emu_st_stance_qp(int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot, const uint32_t* contact,
                     const double* des, const double* kp_linear, const double* gains9, double mass, const double* normals, double* f_body,
                     int32_t* status, double* root_acc, int order_mode) {
  const DevParams P = grf_params();
  StanceGains G;
  for (int i = 0; i < 3; ++i) { G.kd_lin[i] = gains9[i]; G.kp_ang[i] = gains9[3 + i]; G.kd_ang[i] = gains9[6 + i]; }
  G.mass = mass;
  std::vector<int> list((size_t)4 * B, 0);
  int count[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  std::vector<double> rec((size_t)B * STANCE_REC, 0.0);
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, order_mode,
                     [&]() { stance_pack_kernel(B, ld, x0, rot, rot_z, foot, contact, des, kp_linear, G, rec.data(), list.data(), count, f_body, status,
                                                root_acc); });
  run_stance<4>(P, B, rec.data(), contact, list.data(), count, normals, f_body, ld, status, order_mode);
  run_stance<3>(P, B, rec.data(), contact, list.data(), count, normals, f_body, ld, status, order_mode);
  run_stance<2>(P, B, rec.data(), contact, list.data(), count, normals, f_body, ld, status, order_mode);
  run_stance<1>(P, B, rec.data(), contact, list.data(), count, normals, f_body, ld, status, order_mode);
  return 0;
}

// surface_normals_kernel: state [SW_FIELDS][B] (read only), root_pos [3][B] -> normals [12][B]
int emu_st_surface_normals(int B, const double* state, const double* root_pos, double* normals) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0,
                     [&]() { surface_normals_kernel(B, state, root_pos, normals); });
  return 0;
}

}  // extern "C"
