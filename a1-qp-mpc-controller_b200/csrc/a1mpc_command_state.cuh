// a1mpc_command_state.cuh -- the layouts of the IMU and command states and their per-robot start values, for the kernels of
// a1mpc_command.cuh and for the tick's masked reset (a1mpc_tick.cuh).  Defines no kernel, so both translation units may include it.
//
// Both states are batch-major like the swing state (field f of robot b at state[f * B + b]), so a buffer is bound to the B it was
// initialised for.
#pragma once
#include "a1mpc_device.cuh"

namespace a1mpc {

// IMU state (a1mpc_imu_bytes): six MovingWindowFilter(5) (GazeboA1ROS.cpp:100-105, IsaacA1ROS.cpp:62-67), k = acc x,y,z, gyro x,y,z.
// IM_FHDR + 4k + {0,1,2,3}: sum, Neumaier correction, fill count, ring head of filter k;  IM_FVAL + 5k + j: window slot j.
constexpr int IM_WINDOW = 5;
constexpr int IM_FHDR = 0, IM_FVAL = 24;
constexpr int IM_FIELDS = IM_FVAL + 6 * IM_WINDOW;   // 54 doubles per robot

// command state (a1mpc_command_bytes): the adapter's joystick state and the A1CtrlStates fields main_update carries from tick to
// tick, plus the init-time parameters of the robot.
// prev_joy_cmd_ctrl_state is not kept: main_update sets it from joy_cmd_ctrl_state before the toggle and reads it only in the same
// call, so it lives in a register.
constexpr int CM_HEIGHT = 0, CM_CTRL = 1;                    // joy_cmd_body_height, joy_cmd_ctrl_state
constexpr int CM_EUL = 2, CM_POS = 5, CM_KP = 8, CM_LVD = 11;   // root_euler_d[3], root_pos_d[3], kp_linear[3], root_lin_vel_d[3]
constexpr int CM_HMIN = 14, CM_HMAX = 15, CM_LOCK = 16, CM_VARIANT = 18;   // height limits, kp_linear_lock_{x,y}, adapter variant
constexpr int CM_FIELDS = 19;
constexpr int CM_GAZEBO = 0, CM_HARDWARE = 1, CM_ISAAC = 2;   // A1MPC_VARIANT_* of include/a1mpc.h

struct CommandInit {
  double height, hmin, hmax;   // initial joy_cmd_body_height, JOY_CMD_BODY_HEIGHT_MIN / _MAX
  double kp[3], lock[2];       // initial kp_linear, kp_linear_lock_{x,y}
  int variant;
};

// the start values of a1mpc_command_params, as command_init_body takes them
inline CommandInit command_init_params(const a1mpc_command_params& cp) {
  CommandInit P;
  P.height = cp.body_height; P.hmin = cp.body_height_min; P.hmax = cp.body_height_max;
  for (int i = 0; i < 3; ++i) P.kp[i] = cp.kp_linear[i];
  P.lock[0] = cp.kp_linear_lock[0]; P.lock[1] = cp.kp_linear_lock[1];
  P.variant = cp.variant;
  return P;
}

// the per-robot body of imu_init_kernel: empty filters
__device__ __forceinline__ void imu_init_body(int b, int B, double* __restrict__ state) {
  for (int f = 0; f < IM_FIELDS; ++f) state[(size_t)f * B + b] = 0.0;
}

// the per-robot body of command_init_kernel: the adapters' constructor values (GazeboA1ROS.cpp:60-62, GazeboA1ROS.h:130) and
// A1CtrlStates::reset() / resetFromROSParam() (A1CtrlStates.h:35-36, 270-301); ref (may be null) gets the reset values of its nine rows.
__device__ __forceinline__ void command_init_body(int b, int B, const CommandInit& P, double* __restrict__ state, double* __restrict__ ref,
                                                  size_t ref_ld) {
  const size_t lb = (size_t)B;
  double* s = state + b;
  for (int f = 0; f < CM_FIELDS; ++f) s[f * lb] = 0.0;
  s[CM_HEIGHT * lb] = P.height;
  s[CM_HMIN * lb] = P.hmin;
  s[CM_HMAX * lb] = P.hmax;
#pragma unroll
  for (int a = 0; a < 3; ++a) s[(CM_KP + a) * lb] = P.kp[a];
  s[CM_LOCK * lb] = P.lock[0];
  s[(CM_LOCK + 1) * lb] = P.lock[1];
  s[CM_VARIANT * lb] = (double)P.variant;
  if (ref) {
#pragma unroll
    for (int r = 0; r < 9; ++r) ref[r * ref_ld + b] = 0.0;
  }
}

}  // namespace a1mpc
