// emu_swing.cpp -- the swing-leg and terrain-pitch kernels of a1mpc_swing.cuh on the CPU block emulator of cuda_emu.h.
// TEST INFRASTRUCTURE ONLY, next to emu_driver.cpp: the UNCHANGED device code, launched the way a1mpc_api.cu launches it
// (thread per robot, 128-thread blocks).  The state lives on the host here, in the device layout (SW_FIELDS x B doubles).
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

int emu_swing_fields(void) { return SW_FIELDS; }

// a1mpc_swing_init_batch
int emu_swing_init(int B, double* state) {
  launch(B, [&]() { swing_init_kernel(B, state); });
  return 0;
}

// a1mpc_swing_legs_batch (host arrays, ld = B)
int emu_swing_legs(int B, double cps, double dt, const double* kp, const double* kd, double* state, const double* gc, const uint32_t* plan,
                   const double* rot_z, const double* foot_pos_abs, const double* target_rel, const double* foot_force, double* f_kin,
                   uint32_t* contacts, double* cur, double* recent) {
  SwingParams P;
  P.cps = cps; P.dt = dt;
  for (int i = 0; i < 12; ++i) { P.kp[i] = kp[i]; P.kd[i] = kd[i]; }
  launch(B, [&]() { swing_legs_kernel(B, P, state, gc, plan, rot_z, foot_pos_abs, target_rel, foot_force, f_kin, contacts, cur, recent); });
  return 0;
}

// a1mpc_terrain_pitch_batch (host arrays)
int emu_terrain_pitch(int B, double* state, int adapt, const double* root_pos, double* ref, size_t ref_ld, double* pitch) {
  launch(B, [&]() { terrain_pitch_kernel(B, state, adapt, root_pos, ref, ref_ld, pitch); });
  return 0;
}

}  // extern "C"
