// emu_terrain_normals.cpp -- terrain_normals_kernel and terrain_pitch_kernel of a1mpc_swing.cuh, with the swing kernels that fill the
// state they read, on the CPU block emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY: the unchanged device code, launched as
// a1mpc_api.cu launches it (thread per robot, 128-thread blocks), every array dense (ld = B).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_swing.cuh"

using namespace a1mpc;

namespace {
template <class F>
void launch(int B, F&& body) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0, body);
}
}  // namespace

extern "C" {

int emu_tn_swing_fields(void) { return SW_FIELDS; }

int emu_tn_swing_init(int B, double* state) {
  launch(B, [&]() { swing_init_kernel(B, state); });
  return 0;
}

int emu_tn_swing_legs(int B, double cps, double dt, const double* kp, const double* kd, double* state, const double* gc, const uint32_t* plan,
                      const double* rot_z, const double* foot_pos_abs, const double* target_rel, const double* foot_force, double* f_kin,
                      uint32_t* contacts, double* recent) {
  SwingParams P;
  P.cps = cps; P.dt = dt;
  for (int i = 0; i < 12; ++i) { P.kp[i] = kp[i]; P.kd[i] = kd[i]; }
  launch(B, [&]() { swing_legs_kernel(B, P, state, gc, plan, rot_z, foot_pos_abs, target_rel, foot_force, f_kin, contacts, nullptr, recent); });
  return 0;
}

// a1mpc_terrain_pitch_batch (ref [9][ref_ld], pitch may be null)
int emu_tn_terrain_pitch(int B, double* state, int adapt, const double* root_pos, double* ref, size_t ref_ld, double* pitch) {
  launch(B, [&]() { terrain_pitch_kernel(B, state, adapt, root_pos, ref, ref_ld, pitch); });
  return 0;
}

// terrain_normals_kernel: a1mpc_terrain_normals_batch with contacts = sched = NULL, the tick's held pattern with both given
int emu_tn_terrain_normals(int B, double* state, int adapt, const double* root_pos, double* ref, size_t ref_ld, double* pitch, double* normals,
                           const uint32_t* contacts, uint32_t* sched, int N) {
  launch(B, [&]() { terrain_normals_kernel(B, state, adapt, root_pos, ref, ref_ld, pitch, normals, contacts, sched, N); });
  return 0;
}

}  // extern "C"
