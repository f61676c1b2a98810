// a1mpc_command.cu -- launches of the orientation and command stages and of the fused front of a tick (kernels in a1mpc_command.cuh) for
// a1mpc_api.cu.  A translation unit of their own, so that the other kernels of the library compile exactly as they did without them.
#include "a1mpc_internal.h"
#include "a1mpc_command.cuh"

namespace a1mpc {

size_t imu_state_doubles() { return IM_FIELDS; }
size_t command_state_doubles() { return CM_FIELDS; }

cudaError_t imu_init_launch(int B, double* state, cudaStream_t st) {
  imu_init_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, state);
  return cudaGetLastError();
}

cudaError_t orientation_launch(int B, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                               double* euler, double* ang_vel, size_t ld, double* imu_acc, double* imu_ang_vel, cudaStream_t st) {
  orientation_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, quat, gyro, acc, imu, rot, rot_z, euler, ang_vel, ld, imu_acc, imu_ang_vel);
  return cudaGetLastError();
}

cudaError_t command_init_launch(int B, const a1mpc_command_params& cp, double* state, double* ref, size_t ref_ld, cudaStream_t st) {
  command_init_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, command_init_params(cp), state, ref, ref_ld);
  return cudaGetLastError();
}

cudaError_t command_launch(int B, double dt, double* state, const double* cmd, const double* root_pos, size_t pos_ld, uint32_t* movement_mode,
                           double* kp, double* ref, size_t ref_ld, double* des, size_t des_ld, cudaStream_t st) {
  command_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, dt, state, cmd, root_pos, pos_ld, movement_mode, kp, ref, ref_ld, des, des_ld);
  return cudaGetLastError();
}

cudaError_t tick_front_a_launch(int B, double dt, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                                double* x0, double* imu_acc, double* imu_ang_vel, double* cmd_state, const double* cmd, uint32_t* movement_mode,
                                double* kp, double* ref, double* des, cudaStream_t st) {
  const size_t lb = (size_t)B;
  tick_front_a<<<(B + 127) / 128, 128, 0, st>>>(B, dt, quat, gyro, acc, imu, rot, rot_z, x0, x0 + 6 * lb, imu_acc, imu_ang_vel, cmd_state, cmd,
                                                x0 + 3 * lb, movement_mode, kp, ref, des);
  return cudaGetLastError();
}

}  // namespace a1mpc
