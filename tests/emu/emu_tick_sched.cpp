// emu_tick_sched.cpp -- the front kernel of the scheduled tick (tick_front_sched of a1mpc_tick.cuh) and the staged kernels it fuses, on the
// CPU block emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY: the unchanged device code, launched as the library launches it (thread per
// robot, 128-thread blocks), every array dense (ld = B).  The companion of emu_tick.cpp's EMU_TICK_PART 2, with the same flags (tick_sched.mk).
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_tick.cuh"

using namespace a1mpc;

namespace {
template <class F>
void launch(int B, F&& body) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0, body);
}

// gait17: counter_per_gait, counter_per_swing, control_dt, default_foot_pos[12], foot_delta_x_limit, foot_delta_y_limit; N = schedule steps
void params(const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt, int N,
            LegParams& LP, GaitDev& G, SwingParams& SP) {
  for (int i = 0; i < 12; ++i) LP.rho_opt[i] = rho12[i];
  for (int i = 0; i < 20; ++i) LP.rho_fix[i] = rho20[i];
  G.cpg = gait17[0]; G.cps = gait17[1]; G.cdt = gait17[2];
  for (int i = 0; i < 12; ++i) G.dfp[i] = gait17[3 + i];
  G.dxl = gait17[15]; G.dyl = gait17[16]; G.N = N;
  SP.cps = gait17[1]; SP.dt = dt;
  for (int i = 0; i < 12; ++i) { SP.kp[i] = kp12[i]; SP.kd[i] = kd12[i]; }
}
}  // namespace

extern "C" {

int emu_sched_swing_fields(void) { return SW_FIELDS; }

// the staged kernels with update_plan's schedule sched [N][B], then row 0 overwritten by the swing stage's contacts; plan [B] and
// trel [12][B] are the staged path's hand-over arrays.  x0 [12][B]: rows 3-5 (root_pos) and 9-11 (root_lin_vel) read.
int emu_front_sched_staged(int B, const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt,
                           int N, const double* joint_pos, const double* joint_vel, const double* rot, const double* rot_z, const double* x0,
                           const double* lvd, const uint32_t* mode, double* gc, const double* gcs, double* swing, const double* ff, double* fpr,
                           double* jac, double* fvr, double* foot, double* fkin, uint32_t* contacts, uint32_t* sched, uint32_t* plan, double* trel) {
  LegParams LP; GaitDev G; SwingParams SP;
  params(rho12, rho20, gait17, kp12, kd12, dt, N, LP, G, SP);
  const size_t lb = (size_t)B;
  launch(B, [&]() { leg_kinematics_kernel(B, joint_pos, joint_vel, rot, LP, fpr, jac, fvr, foot, nullptr); });
  launch(B, [&]() {
    update_plan_kernel(B, G, gc, gcs, mode, x0 + 9 * lb, lvd, rot_z, rot, x0 + 3 * lb, plan, sched, trel, nullptr, nullptr);
  });
  launch(B, [&]() { swing_legs_kernel(B, SP, swing, gc, plan, rot_z, foot, trel, ff, fkin, contacts, nullptr, nullptr); });
  for (int b = 0; b < B; ++b) sched[b] = contacts[b];
  return 0;
}

int emu_front_sched_fused(int B, const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12, double dt,
                          int N, const double* joint_pos, const double* joint_vel, const double* rot, const double* rot_z, const double* x0,
                          const double* lvd, const uint32_t* mode, double* gc, const double* gcs, double* swing, const double* ff, double* fpr,
                          double* jac, double* fvr, double* foot, double* fkin, uint32_t* contacts, uint32_t* sched) {
  LegParams LP; GaitDev G; SwingParams SP;
  params(rho12, rho20, gait17, kp12, kd12, dt, N, LP, G, SP);
  launch(B, [&]() {
    tick_front_sched(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts, sched);
  });
  return 0;
}

}  // extern "C"
