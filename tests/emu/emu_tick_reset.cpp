// emu_tick_reset.cpp -- the masked reset kernels of a control tick (tick_reset_robots_kernel, ekf_init_pending of a1mpc_tick.cuh) and the
// init kernels of the whole batch they must agree with, on the CPU block emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY: the unchanged
// device code, launched as the library launches it (thread per robot, 128-thread blocks), every array dense (ld = B).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_command.cuh"
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_tick.cuh"

using namespace a1mpc;

namespace {
template <class F>
void launch(int B, F&& body) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0, body);
}

CommandInit cinit(int variant, const double* hp3, const double* kp3, const double* lock2) {
  CommandInit P;
  P.height = hp3[0]; P.hmin = hp3[1]; P.hmax = hp3[2];
  for (int i = 0; i < 3; ++i) P.kp[i] = kp3[i];
  P.lock[0] = lock2[0]; P.lock[1] = lock2[1];
  P.variant = variant;
  return P;
}
}  // namespace

extern "C" {

// IM_FIELDS, CM_FIELDS, SW_FIELDS, EKF_STATE_DOUBLES, WARM_HDR
void emu_reset_sizes(int* out) {
  const int v[5] = {IM_FIELDS, CM_FIELDS, SW_FIELDS, EKF_STATE_DOUBLES, WARM_HDR};
  for (int i = 0; i < 5; ++i) out[i] = v[i];
}

// hp3: body_height, body_height_min, body_height_max.  imu, ref, warm and pending may be null.
int emu_tick_reset_robots(int B, const uint8_t* mask, int variant, const double* hp3, const double* kp3, const double* lock2, double* x0, double* gc,
                          double* tau, double* imu, double* cmd, double* ref, double* swing, uint32_t* warm, int warm_words, uint8_t* pending) {
  const CommandInit P = cinit(variant, hp3, kp3, lock2);
  launch(B, [&]() { tick_reset_robots_kernel(B, mask, P, x0, gc, tau, imu, cmd, ref, swing, warm, warm_words, pending); });
  return 0;
}

// the whole-batch init kernels of a1mpc_tick_reset (imu may be null)
int emu_init_kernels(int B, int variant, const double* hp3, const double* kp3, const double* lock2, double* imu, double* cmd, double* ref,
                     double* swing) {
  const CommandInit P = cinit(variant, hp3, kp3, lock2);
  if (imu) launch(B, [&]() { imu_init_kernel(B, imu); });
  launch(B, [&]() { command_init_kernel(B, P, cmd, ref, (size_t)B); });
  launch(B, [&]() { swing_init_kernel(B, swing); });
  return 0;
}

int emu_ekf_init(int B, double* state, const double* fpr, const double* rot) {
  launch(B, [&]() { ekf_init_kernel(B, state, fpr, rot); });
  return 0;
}

int emu_ekf_init_pending(int B, uint8_t* pending, double* state, const double* fpr, const double* rot, double* x0) {
  launch(B, [&]() { ekf_init_pending(B, pending, state, fpr, rot, x0); });
  return 0;
}

}  // extern "C"
