// emu_tick.cpp -- the fused kernels of a control tick (tick_front_a of a1mpc_command.cuh, tick_front_b of a1mpc_tick.cuh) and the staged
// kernels they fuse, on the CPU block emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY: the unchanged device code, launched as the library
// launches it (thread per robot, 128-thread blocks), every array dense (ld = B).  Compiled twice (tick.mk): EMU_TICK_PART 1 = the front
// (orientation, command), 2 = the middle (kinematics, update_plan, swing legs).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#if EMU_TICK_PART == 1
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_command.cuh"
#else
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_tick.cuh"
#endif

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

#if EMU_TICK_PART == 1
// x0 [12][B]: rows 0-2 and 6-8 written, rows 3-5 read (root_pos); imu and ref may be null
int emu_front_a_staged(int B, double dt, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                       double* x0, double* imu_acc, double* imu_ang_vel, double* cmd_state, const double* cmd, uint32_t* mode, double* kp,
                       double* ref, double* des) {
  const size_t lb = (size_t)B;
  launch(B, [&]() { orientation_kernel(B, quat, gyro, acc, imu, rot, rot_z, x0, x0 + 6 * lb, lb, imu_acc, imu_ang_vel); });
  launch(B, [&]() { command_kernel(B, dt, cmd_state, cmd, x0 + 3 * lb, lb, mode, kp, ref, lb, des, lb); });
  return 0;
}

int emu_front_a_fused(int B, double dt, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                      double* x0, double* imu_acc, double* imu_ang_vel, double* cmd_state, const double* cmd, uint32_t* mode, double* kp,
                      double* ref, double* des) {
  const size_t lb = (size_t)B;
  launch(B, [&]() {
    tick_front_a(B, dt, quat, gyro, acc, imu, rot, rot_z, x0, x0 + 6 * lb, imu_acc, imu_ang_vel, cmd_state, cmd, x0 + 3 * lb, mode, kp, ref, des);
  });
  return 0;
}
#else
int emu_swing_fields(void) { return SW_FIELDS; }

namespace {
void params(const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt, LegParams& LP,
            GaitDev& G, SwingParams& SP) {
  for (int i = 0; i < 12; ++i) LP.rho_opt[i] = rho12[i];
  for (int i = 0; i < 20; ++i) LP.rho_fix[i] = rho20[i];
  // gait17: counter_per_gait, counter_per_swing, control_dt, default_foot_pos[12], foot_delta_x_limit, foot_delta_y_limit
  G.cpg = gait17[0]; G.cps = gait17[1]; G.cdt = gait17[2];
  for (int i = 0; i < 12; ++i) G.dfp[i] = gait17[3 + i];
  G.dxl = gait17[15]; G.dyl = gait17[16]; G.N = 0;
  SP.cps = gait17[1]; SP.dt = dt;
  for (int i = 0; i < 12; ++i) { SP.kp[i] = kp12[i]; SP.kd[i] = kd12[i]; }
}
}  // namespace

// x0 [12][B]: rows 3-5 (root_pos) and 9-11 (root_lin_vel) read; plan [B] and trel [12][B] are the staged path's hand-over arrays
int emu_front_b_staged(int B, const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt,
                       const double* joint_pos, const double* joint_vel, const double* rot, const double* rot_z, const double* x0, const double* lvd,
                       const uint32_t* mode, double* gc, const double* gcs, double* swing, const double* ff, double* fpr, double* jac, double* fvr,
                       double* foot, double* fkin, uint32_t* contacts, uint32_t* plan, double* trel) {
  LegParams LP; GaitDev G; SwingParams SP;
  params(rho12, rho20, gait17, kp12, kd12, dt, LP, G, SP);
  const size_t lb = (size_t)B;
  launch(B, [&]() { leg_kinematics_kernel(B, joint_pos, joint_vel, rot, LP, fpr, jac, fvr, foot, nullptr); });
  launch(B, [&]() {
    update_plan_kernel(B, G, gc, gcs, mode, x0 + 9 * lb, lvd, rot_z, rot, x0 + 3 * lb, plan, nullptr, trel, nullptr, nullptr);
  });
  launch(B, [&]() { swing_legs_kernel(B, SP, swing, gc, plan, rot_z, foot, trel, ff, fkin, contacts, nullptr, nullptr); });
  return 0;
}

int emu_front_b_fused(int B, const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt,
                      const double* joint_pos, const double* joint_vel, const double* rot, const double* rot_z, const double* x0, const double* lvd,
                      const uint32_t* mode, double* gc, const double* gcs, double* swing, const double* ff, double* fpr, double* jac, double* fvr,
                      double* foot, double* fkin, uint32_t* contacts) {
  LegParams LP; GaitDev G; SwingParams SP;
  params(rho12, rho20, gait17, kp12, kd12, dt, LP, G, SP);
  launch(B, [&]() {
    tick_front_b(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts);
  });
  return 0;
}
#endif

}  // extern "C"
