// a1mpc_command.cuh -- the first two stages of a control tick, batched, with the adapters' own state on the device:
//   * the orientation stage of the robot adapters (GazeboA1ROS.cpp:235-299, HardwareA1ROS.cpp:262-276, IsaacA1ROS.cpp:183-241):
//     root_rot_mat = root_quat.toRotationMatrix(), root_euler = Utils::quat_to_euler(root_quat) (utils/Utils.cpp:7-32),
//     root_rot_mat_z = AngleAxisd(yaw, UnitZ), root_ang_vel = root_rot_mat * imu_ang_vel, with the 5-sample MovingWindowFilters
//     of the Gazebo / Isaac IMU callbacks in front
//   * the command stage, main_update's front half (GazeboA1ROS.cpp:117-188, HardwareA1ROS.cpp:98-158, IsaacA1ROS.cpp:75-137):
//     body height, walking toggle, desired velocities and euler angles, movement_mode, xy position lock
// Include from exactly one translation unit (a1mpc_command.cu) -- and from tests/emu (g++, A1MPC_EMU).
//
// The layouts of both states and their start values are in a1mpc_command_state.cuh.  One thread per robot: a few dozen flops over a
// few dozen doubles, every load and store coalesced.
#pragma once
#include "a1mpc_command_state.cuh"
#include "a1mpc_filter.cuh"

namespace a1mpc {

__global__ void imu_init_kernel(int B, double* __restrict__ state) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  imu_init_body(b, B, state);
}

// one IMU sample and one pose per robot, thread per robot.  quat [4][B] (w, x, y, z), gyro / acc [3][B] and imu_acc / imu_ang_vel
// [3][B] have leading dimension B; rot, rot_z [9][B], euler and ang_vel [3][B] (rows 0-2 and 6-8 of x0) leading dimension ld.  imu
// (the filter state), acc and every output may be null.
// the per-robot body of orientation_kernel, shared with tick_front_a
__device__ __forceinline__ void orientation_body(int b, int B, const double* __restrict__ quat, const double* __restrict__ gyro,
                                                 const double* __restrict__ acc, double* __restrict__ imu, double* __restrict__ rot,
                                                 double* __restrict__ rot_z, double* __restrict__ euler, double* __restrict__ ang_vel, size_t ld,
                                                 double* __restrict__ imu_acc, double* __restrict__ imu_ang_vel) {
  const size_t lb = (size_t)B;
  double* s = imu ? imu + b : nullptr;
  // imu_callback (GazeboA1ROS.cpp:282-299, IsaacA1ROS.cpp:224-241): filter k of window 5, or the raw sample (HardwareA1ROS.cpp:273-274)
  double g[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double v = gyro[a * lb + b];
    if (s) v = mw_filter(s, lb, IM_WINDOW, IM_FVAL + IM_WINDOW * (3 + a), IM_FHDR + 4 * (3 + a), v);
    g[a] = v;
    if (imu_ang_vel) imu_ang_vel[a * lb + b] = v;
  }
  if (acc) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      double v = acc[a * lb + b];
      if (s) v = mw_filter(s, lb, IM_WINDOW, IM_FVAL + IM_WINDOW * a, IM_FHDR + 4 * a, v);
      if (imu_acc) imu_acc[a * lb + b] = v;
    }
  }
  const double w = quat[b], x = quat[lb + b], y = quat[2 * lb + b], z = quat[3 * lb + b];   // used as given: no normalisation
  // Eigen's QuaternionBase::toRotationMatrix
  const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  const double R[9] = {1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1.0 - (txx + tyy)};
  if (rot) {
#pragma unroll
    for (int k = 0; k < 9; ++k) rot[k * ld + b] = R[k];
  }
  // Utils::quat_to_euler (utils/Utils.cpp:7-32): roll, pitch (t2 clamped to +-1), yaw
  const double ysq = y * y;
  const double t0 = 2.0 * (w * x + y * z), t1 = 1.0 - 2.0 * (x * x + ysq);
  double t2 = 2.0 * (w * y - z * x);
  t2 = t2 > 1.0 ? 1.0 : t2;
  t2 = t2 < -1.0 ? -1.0 : t2;
  const double t3 = 2.0 * (w * z + x * y), t4 = 1.0 - 2.0 * (ysq + z * z);
  const double yaw = atan2(t3, t4);
  if (euler) {
    euler[b] = atan2(t0, t1);
    euler[ld + b] = asin(t2);
    euler[2 * ld + b] = yaw;
  }
  // Eigen's AngleAxis::toRotationMatrix about UnitZ: cos / sin of the full angle, diagonal (1 - c) * axis .* axis + c
  if (rot_z) {
    double sn, c;
    sincos(yaw, &sn, &c);
    const double Z[9] = {c, 0.0 - sn, 0.0, 0.0 + sn, c, 0.0, 0.0, 0.0, (1.0 - c) + c};
#pragma unroll
    for (int k = 0; k < 9; ++k) rot_z[k * ld + b] = Z[k];
  }
  // root_ang_vel = root_rot_mat * imu_ang_vel with the rotation of this call
  if (ang_vel) {
#pragma unroll
    for (int i = 0; i < 3; ++i) ang_vel[i * ld + b] = R[3 * i] * g[0] + R[3 * i + 1] * g[1] + R[3 * i + 2] * g[2];
  }
}

__global__ void orientation_kernel(int B, const double* __restrict__ quat, const double* __restrict__ gyro, const double* __restrict__ acc,
                                   double* __restrict__ imu, double* __restrict__ rot, double* __restrict__ rot_z, double* __restrict__ euler,
                                   double* __restrict__ ang_vel, size_t ld, double* __restrict__ imu_acc, double* __restrict__ imu_ang_vel) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  orientation_body(b, B, quat, gyro, acc, imu, rot, rot_z, euler, ang_vel, ld, imu_acc, imu_ang_vel);
}

__global__ void command_init_kernel(int B, CommandInit P, double* __restrict__ state, double* __restrict__ ref, size_t ref_ld) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  command_init_body(b, B, P, state, ref, ref_ld);
}

// main_update's front half (GazeboA1ROS.cpp:122-188; HardwareA1ROS.cpp:104-158; IsaacA1ROS.cpp:81-137), thread per robot.
// cmd [7][B]: velx, vely, velz, roll rate, pitch rate, yaw rate, toggle request.  root_pos [3][pos_ld]; kp [3][des_ld], des [12][des_ld]
// (may be null), ref [9][ref_ld] (may be null: then root_euler_d[1] comes from the state).
// the per-robot body of command_kernel, shared with tick_front_a
__device__ __forceinline__ void command_body(int b, int B, double dt, double* __restrict__ state, const double* __restrict__ cmd,
                                             const double* __restrict__ root_pos, size_t pos_ld, uint32_t* __restrict__ movement_mode,
                                             double* __restrict__ kp, double* __restrict__ ref, size_t ref_ld, double* __restrict__ des, size_t des_ld) {
  const size_t lb = (size_t)B;
  double* s = state + b;
  double c[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) c[k] = cmd[k * lb + b];
  const int variant = (int)s[CM_VARIANT * lb];
  const bool hw = variant == CM_HARDWARE;
  // body height integrated and clamped (:122-130)
  double h = s[CM_HEIGHT * lb] + c[2] * dt;
  if (h >= s[CM_HMAX * lb]) h = s[CM_HMAX * lb];
  if (h <= s[CM_HMIN * lb]) h = s[CM_HMIN * lb];
  // walking toggle (:140-147)
  const int prev = (int)s[CM_CTRL * lb];
  int ctrl = prev;
  if (c[6] != 0.0) ctrl = (ctrl + 1) % 2;
  // desired velocities (:149-157).  Only Gazebo sets root_lin_vel_d[2] = velz (GazeboA1ROS.cpp:152); the hardware and Isaac
  // adapters set x and y only (HardwareA1ROS.cpp:121-123, IsaacA1ROS.cpp:99-101) and leave z at its reset value
  double lvd[3] = {c[0], c[1], variant == CM_GAZEBO ? c[2] : s[(CM_LVD + 2) * lb]};
  // desired euler angles (:158-160).  root_euler_d[1] starts from row 1 of ref when given: compute_grf's terrain adaptation
  // overwrites it there (A1RobotControl.cpp:358-364) and the next tick integrates on top of that value.  The hardware adapter
  // assigns the roll and pitch rates themselves (HardwareA1ROS.cpp:129-130).
  double e[3], p[3], k[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) { e[a] = s[(CM_EUL + a) * lb]; p[a] = s[(CM_POS + a) * lb]; k[a] = s[(CM_KP + a) * lb]; }
  if (ref) e[1] = ref[ref_ld + b];
  if (hw) {
    e[0] = c[3];
    e[1] = c[4];
  } else {
    e[0] += c[3] * dt;
    e[1] += c[4] * dt;
  }
  e[2] += c[5] * dt;
  p[2] = h;
  // movement mode and the xy position lock (:163-188)
  uint32_t mode = 0;
  if (ctrl == 1) {
    mode = 1;
  } else if (ctrl == 0 && prev == 1) {
    p[0] = root_pos[b]; p[1] = root_pos[pos_ld + b];
    k[0] = s[CM_LOCK * lb]; k[1] = s[(CM_LOCK + 1) * lb];
  }
  if (mode == 1) {
    if (sqrt(lvd[0] * lvd[0] + lvd[1] * lvd[1]) > 0.05) {
      p[0] = root_pos[b]; p[1] = root_pos[pos_ld + b];
      k[0] = 0.0; k[1] = 0.0;
    } else {
      k[0] = s[CM_LOCK * lb]; k[1] = s[(CM_LOCK + 1) * lb];
    }
  }
  s[CM_HEIGHT * lb] = h;
  s[CM_CTRL * lb] = (double)ctrl;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    s[(CM_EUL + a) * lb] = e[a]; s[(CM_POS + a) * lb] = p[a]; s[(CM_KP + a) * lb] = k[a]; s[(CM_LVD + a) * lb] = lvd[a];
    kp[a * des_ld + b] = k[a];
  }
  movement_mode[b] = mode;
  if (ref) {   // root_euler_d[0..1], root_ang_vel_d, root_lin_vel_d (body), root_pos_d[2]
    const double r[9] = {e[0], e[1], c[3], c[4], c[5], lvd[0], lvd[1], lvd[2], p[2]};
#pragma unroll
    for (int i = 0; i < 9; ++i) ref[i * ref_ld + b] = r[i];
  }
  if (des) {   // root_euler_d, root_pos_d, root_lin_vel_d (body), root_ang_vel_d
    const double d[12] = {e[0], e[1], e[2], p[0], p[1], p[2], lvd[0], lvd[1], lvd[2], c[3], c[4], c[5]};
#pragma unroll
    for (int i = 0; i < 12; ++i) des[i * des_ld + b] = d[i];
  }
}

__global__ void command_kernel(int B, double dt, double* __restrict__ state, const double* __restrict__ cmd, const double* __restrict__ root_pos,
                               size_t pos_ld, uint32_t* __restrict__ movement_mode, double* __restrict__ kp, double* __restrict__ ref, size_t ref_ld,
                               double* __restrict__ des, size_t des_ld) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  command_body(b, B, dt, state, cmd, root_pos, pos_ld, movement_mode, kp, ref, ref_ld, des, des_ld);
}

// The front of a control tick (a1mpc_tick_run), thread per robot: orientation_body then command_body, every array dense (ld = B).  The
// command stage reads none of the orientation stage's outputs (root_pos is the previous tick's estimate), so the pair is the two
// staged kernels back to back; this translation unit's --fmad=false keeps each stage's rounding what it is alone.
__global__ void tick_front_a(int B, double dt, const double* __restrict__ quat, const double* __restrict__ gyro, const double* __restrict__ acc,
                             double* __restrict__ imu, double* __restrict__ rot, double* __restrict__ rot_z, double* __restrict__ euler,
                             double* __restrict__ ang_vel, double* __restrict__ imu_acc, double* __restrict__ imu_ang_vel,
                             double* __restrict__ cmd_state, const double* __restrict__ cmd, const double* __restrict__ root_pos,
                             uint32_t* __restrict__ movement_mode, double* __restrict__ kp, double* __restrict__ ref, double* __restrict__ des) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t lb = (size_t)B;
  orientation_body(b, B, quat, gyro, acc, imu, rot, rot_z, euler, ang_vel, lb, imu_acc, imu_ang_vel);
  command_body(b, B, dt, cmd_state, cmd, root_pos, lb, movement_mode, kp, ref, lb, des, lb);
}

}  // namespace a1mpc
