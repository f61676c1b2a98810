// emu_gait.cpp -- the per-robot gait kernels of a1mpc_gait.cuh and the plain kernels they must reproduce with trot rows, on the CPU block
// emulator of cuda_emu.h.  TEST INFRASTRUCTURE ONLY: the unchanged device code, launched as the library launches it (thread per robot,
// 128-thread blocks), every array dense (ld = B).
#define A1MPC_EMU 1
#include "cuda_emu.h"

// the row check's atomicMin on one 64-bit word (cuda_emu.h has the 32-bit atomicAdd only)
inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long cur = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < cur && !__atomic_compare_exchange_n(p, &cur, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return cur;
}

using std::isfinite;   // the device isfinite of the row check
#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_gait.cuh"

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

int emu_gait_swing_fields(void) { return SW_FIELDS; }

// the tick's front stage.  kind 0: tick_front_b / tick_front_sched (gait ignored); 1: their gait twins; 2: the staged gait kernels
// (leg_kinematics_kernel, update_plan_gait_kernel, swing_legs_gait_kernel, schedule row 0 = the swing stage's contacts), with plan [B]
// and trel [12][B] their hand-over.  N = 0: no schedule (sched may be NULL).
int emu_gait_front(int kind, int B, const double* rho12, const double* rho20, const double* gait17, const double* kp12, const double* kd12,
                   double dt, int N, const double* gait, const double* joint_pos, const double* joint_vel, const double* rot, const double* rot_z,
                   const double* x0, const double* lvd, const uint32_t* mode, double* gc, const double* gcs, double* swing, const double* ff,
                   double* fpr, double* jac, double* fvr, double* foot, double* fkin, uint32_t* contacts, uint32_t* sched, uint32_t* plan,
                   double* trel) {
  LegParams LP; GaitDev G; SwingParams SP;
  params(rho12, rho20, gait17, kp12, kd12, dt, N, LP, G, SP);
  const size_t lb = (size_t)B;
  if (kind == 0 && N > 0)
    launch(B, [&]() { tick_front_sched(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts, sched); });
  else if (kind == 0)
    launch(B, [&]() { tick_front_b(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts); });
  else if (kind == 1 && N > 0)
    launch(B, [&]() {
      tick_front_sched_gait(B, LP, G, SP, gait, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts, sched);
    });
  else if (kind == 1)
    launch(B, [&]() { tick_front_b_gait(B, LP, G, SP, gait, joint_pos, joint_vel, rot, rot_z, x0, lvd, mode, gc, gcs, swing, ff, fpr, jac, fvr, foot, fkin, contacts); });
  else {
    launch(B, [&]() { leg_kinematics_kernel(B, joint_pos, joint_vel, rot, LP, fpr, jac, fvr, foot, nullptr); });
    launch(B, [&]() {
      update_plan_gait_kernel(B, G, gait, gc, gcs, mode, x0 + 9 * lb, lvd, rot_z, rot, x0 + 3 * lb, plan, N > 0 ? sched : nullptr, trel, nullptr, nullptr);
    });
    launch(B, [&]() { swing_legs_gait_kernel(B, SP, gait, swing, gc, plan, rot_z, foot, trel, ff, fkin, contacts, nullptr, nullptr); });
    if (N > 0)
      for (int b = 0; b < B; ++b) sched[b] = contacts[b];
  }
  return 0;
}

// update_plan_kernel (gait NULL) or update_plan_gait_kernel, every output
int emu_gait_update_plan(int B, const double* gait17, int N, const double* gait, double* gc, const double* gcs, const uint32_t* mode, const double* lv,
                         const double* lvd, const double* rz, const double* rot, const double* pos, uint32_t* plan, uint32_t* sched, double* t_rel,
                         double* t_abs, double* t_world) {
  const double zero[32] = {0};
  LegParams LP; GaitDev G; SwingParams SP;
  params(zero, zero, gait17, zero, zero, 1.0, N, LP, G, SP);
  if (gait)
    launch(B, [&]() { update_plan_gait_kernel(B, G, gait, gc, gcs, mode, lv, lvd, rz, rot, pos, plan, sched, t_rel, t_abs, t_world); });
  else
    launch(B, [&]() { update_plan_kernel(B, G, gc, gcs, mode, lv, lvd, rz, rot, pos, plan, sched, t_rel, t_abs, t_world); });
  return 0;
}

// swing_legs_kernel (gait NULL, cps from gait17) or swing_legs_gait_kernel
int emu_gait_swing_legs(int B, const double* gait17, const double* kp12, const double* kd12, double dt, const double* gait, double* swing,
                        const double* gc, const uint32_t* plan, const double* rz, const double* fpa, const double* tgt, const double* ff, double* fkin,
                        uint32_t* contacts, double* cur, double* rc) {
  const double zero[32] = {0};
  LegParams LP; GaitDev G; SwingParams SP;
  params(zero, zero, gait17, kp12, kd12, dt, 0, LP, G, SP);
  if (gait)
    launch(B, [&]() { swing_legs_gait_kernel(B, SP, gait, swing, gc, plan, rz, fpa, tgt, ff, fkin, contacts, cur, rc); });
  else
    launch(B, [&]() { swing_legs_kernel(B, SP, swing, gc, plan, rz, fpa, tgt, ff, fkin, contacts, cur, rc); });
  return 0;
}

// gait_check_kernel: the least (b << 2 | rule) over the bad rows, all ones when every row is valid
unsigned long long emu_gait_check(int B, const double* gait) {
  unsigned long long bad = ~0ull;
  launch(B, [&]() { gait_check_kernel(B, gait, &bad); });
  return bad;
}

}  // extern "C"
