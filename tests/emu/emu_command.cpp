// emu_command.cpp -- the orientation and command kernels of a1mpc_command.cuh on the CPU block emulator of cuda_emu.h.
// TEST INFRASTRUCTURE ONLY, next to emu_swing.cpp: the UNCHANGED device code, launched the way a1mpc_command.cu launches it
// (thread per robot, 128-thread blocks).  The states live on the host here, in the device layout (fields x B doubles).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_command.cuh"

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

int emu_imu_fields(void) { return IM_FIELDS; }
int emu_command_fields(void) { return CM_FIELDS; }

int emu_imu_init(int B, double* state) {
  launch(B, [&]() { imu_init_kernel(B, state); });
  return 0;
}

// a1mpc_orientation_batch (host arrays; rot, rot_z, euler, ang_vel with leading dimension ld)
int emu_orientation(int B, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z, double* euler,
                    double* ang_vel, size_t ld, double* imu_acc, double* imu_ang_vel) {
  launch(B, [&]() { orientation_kernel(B, quat, gyro, acc, imu, rot, rot_z, euler, ang_vel, ld, imu_acc, imu_ang_vel); });
  return 0;
}

int emu_command_init(int B, int variant, double height, double hmin, double hmax, const double* kp3, const double* lock2, double* state,
                     double* ref, size_t ref_ld) {
  CommandInit P;
  P.height = height; P.hmin = hmin; P.hmax = hmax;
  for (int i = 0; i < 3; ++i) P.kp[i] = kp3[i];
  P.lock[0] = lock2[0]; P.lock[1] = lock2[1];
  P.variant = variant;
  launch(B, [&]() { command_init_kernel(B, P, state, ref, ref_ld); });
  return 0;
}

int emu_command(int B, double dt, double* state, const double* cmd, const double* root_pos, size_t pos_ld, uint32_t* mode, double* kp,
                double* ref, size_t ref_ld, double* des, size_t des_ld) {
  launch(B, [&]() { command_kernel(B, dt, state, cmd, root_pos, pos_ld, mode, kp, ref, ref_ld, des, des_ld); });
  return 0;
}

}  // extern "C"
