// a1mpc_tick.cuh -- the middle of a control tick (a1mpc_tick_run) in one kernel (tick_front_b, or tick_front_sched in the scheduled tick):
// leg kinematics, update_plan and generate_swing_legs_ctrl in one thread per robot, from the per-robot bodies of leg_kinematics_kernel,
// update_plan_kernel and swing_legs_kernel.
// Include from exactly one translation unit (a1mpc_api.cu) -- and from tests/emu (g++, A1MPC_EMU).
//
// What crosses a stage boundary in registers instead of memory: foot_pos_abs (kinematics -> swing), plan_contacts and foot_pos_target_rel
// (update_plan -> swing).  Neither of the latter two is stored.  tick_front_b computes no contact schedule; tick_front_sched, the same body,
// also writes the schedule of the scheduled tick.  The stored outputs are the ones later
// stages read: foot_pos_rel, foot_vel_rel and jac (EKF, torques), foot_pos_abs (the solve's foot), f_kin and contacts (solve, torques), and
// the gait counters and swing state (next tick).
// Also the two kernels of a per-robot reset (a1mpc_tick_reset_robots): tick_reset_robots_kernel, and ekf_init_pending in the next run.
// Bit-identity with the staged kernels: the compiler contracts products into FMAs per kernel, so every stage keeps the loop shape it has
// in its own kernel.  The foothold targets and the swing legs run in one rolled leg loop, as both do in update_plan_kernel and
// swing_legs_kernel: unrolled, the foothold's loop-invariant product kf * (v - vd) is no longer hoisted and the other product of dx / dy gets
// contracted, which moves the targets by an ulp.  The loop index then selects each leg's registers instead of indexing an array, which would
// go to local memory.
#pragma once
#include "a1mpc_command_state.cuh"
#include "a1mpc_estim.cuh"
#include "a1mpc_misc.cuh"
#include "a1mpc_swing.cuh"

namespace a1mpc {

// value i of four held in registers, for an index the rolled leg loop does not know at compile time
__device__ __forceinline__ double leg_select(double v0, double v1, double v2, double v3, int i) {
  return i == 0 ? v0 : (i == 1 ? v1 : (i == 2 ? v2 : v3));
}

// the swing stage's inputs as tick_front_b holds them: the gait counters from memory (this thread has just written them), the planned
// contacts, this leg's foothold target and the four feet's foot_pos_abs in registers (the leg's three selected by the loop index)
struct SwingSrcTick {
  const double* gc;
  uint32_t pl;
  const double (&fpa)[12];
  const double (&tgt)[3];
  size_t ld;
  int b;
  __device__ __forceinline__ uint32_t plan() const { return pl; }
  __device__ __forceinline__ double g(int i) const { return gc[(size_t)i * ld + b]; }
  __device__ __forceinline__ double p(int i, int a) const { return leg_select(fpa[a], fpa[3 + a], fpa[6 + a], fpa[9 + a], i); }
  __device__ __forceinline__ double fin(int, int a) const { return tgt[a]; }
};

// the body of both kernels below; sched == nullptr (tick_front_b) computes no schedule.  every array dense (ld = B).  x0 [12][B]: rows 3-5
// (root_pos) and 9-11 (root_lin_vel) read; lin_vel_d [3][B] is ref + 5 B (MPC mode) or des + 6 B (QP mode).
__device__ __forceinline__ void tick_front_b_body(int B, const LegParams& LP, const GaitDev& G, const SwingParams& SP, const double* __restrict__ joint_pos,
                                                  const double* __restrict__ joint_vel, const double* __restrict__ rot, const double* __restrict__ rot_z,
                                                  const double* __restrict__ x0, const double* __restrict__ lin_vel_d, const uint32_t* __restrict__ mode,
                                                  double* __restrict__ gc, const double* __restrict__ gcs, double* __restrict__ swing_state,
                                                  const double* __restrict__ foot_force, double* __restrict__ fpr, double* __restrict__ jac,
                                                  double* __restrict__ fvr, double* __restrict__ foot, double* __restrict__ fkin,
                                                  uint32_t* __restrict__ contacts, uint32_t* __restrict__ sched) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  // leg kinematics
  double fpa[12];
  leg_kinematics_body(b, ld, joint_pos, joint_vel, rot, LP, fpr, jac, fvr, foot, nullptr, [&](int k, double v) { fpa[k] = v; });
  // update_plan: gait counters and planned contacts; schedule rows 1 .. N-1 (row 0 waits for the swing stage's contacts)
  double c[4], sp[4];
  const bool walk = mode[b] != 0;
  const uint32_t plan = update_plan_counters(b, ld, G, gc, gcs, walk, c, sp);
  if (sched) update_plan_sched(b, ld, G, walk, c, sp, 1, sched);
  PlanTargets T;
  plan_targets_setup(b, ld, G, x0 + 9 * ld, lin_vel_d, rot_z, rot, x0 + 3 * ld, T);
  // swing legs (swing_legs_kernel's body), each leg right after its foothold target, in the same rolled leg loops as the staged kernels
  double* s = swing_state + b;
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = rot_z[(size_t)k * ld + b];
  uint32_t early = (uint32_t)s[(size_t)SW_EARLY * ld];
  uint32_t cm = 0;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    double f[3];
    plan_target_leg(i, G, leg_select(sp[0], sp[1], sp[2], sp[3], i), T, f);
    const SwingSrcTick src{gc, plan, fpa, f, ld, b};
    swing_leg(i, b, ld, SP, s, R, plan, early, cm, src, foot_force, fkin, nullptr, nullptr);
  }
  s[(size_t)SW_EARLY * ld] = (double)early;
  contacts[b] = cm;
  if (sched) sched[b] = cm;
}

// the held-pattern tick (gait.horizon = 0): no schedule
__global__ void tick_front_b(int B, LegParams LP, GaitDev G, SwingParams SP, const double* __restrict__ joint_pos, const double* __restrict__ joint_vel,
                             const double* __restrict__ rot, const double* __restrict__ rot_z, const double* __restrict__ x0,
                             const double* __restrict__ lin_vel_d, const uint32_t* __restrict__ mode, double* __restrict__ gc,
                             const double* __restrict__ gcs, double* __restrict__ swing_state, const double* __restrict__ foot_force,
                             double* __restrict__ fpr, double* __restrict__ jac, double* __restrict__ fvr, double* __restrict__ foot,
                             double* __restrict__ fkin, uint32_t* __restrict__ contacts) {
  tick_front_b_body(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lin_vel_d, mode, gc, gcs, swing_state, foot_force, fpr, jac, fvr, foot, fkin,
                    contacts, nullptr);
}

// the scheduled tick (gait.horizon = N = G.N): tick_front_b plus the contact schedule sched [N][B] the solve takes.  Rows 1 .. N-1 are
// update_plan's; row 0 is the swing stage's contacts (plan OR early contact), so the solve's first step stands on the feet the torque stage
// treats as stance.
__global__ void tick_front_sched(int B, LegParams LP, GaitDev G, SwingParams SP, const double* __restrict__ joint_pos, const double* __restrict__ joint_vel,
                                 const double* __restrict__ rot, const double* __restrict__ rot_z, const double* __restrict__ x0,
                                 const double* __restrict__ lin_vel_d, const uint32_t* __restrict__ mode, double* __restrict__ gc,
                                 const double* __restrict__ gcs, double* __restrict__ swing_state, const double* __restrict__ foot_force,
                                 double* __restrict__ fpr, double* __restrict__ jac, double* __restrict__ fvr, double* __restrict__ foot,
                                 double* __restrict__ fkin, uint32_t* __restrict__ contacts, uint32_t* __restrict__ sched) {
  tick_front_b_body(B, LP, G, SP, joint_pos, joint_vel, rot, rot_z, x0, lin_vel_d, mode, gc, gcs, swing_state, foot_force, fpr, jac, fvr, foot, fkin,
                    contacts, sched);
}

// a1mpc_tick_reset_robots: robot b with mask[b] != 0 gets the start values a1mpc_tick_reset writes (zero x0, gait counters, tau and warm
// slot; the bodies of imu_init_kernel, command_init_kernel and swing_init_kernel), and pending[b] = 1 so that the next run initialises its
// EKF (ekf_init_pending).  imu, ref, warm and pending may be null.  Thread per robot: the warp reads 32 mask bytes at once and every
// batch-major store of a fully masked warp is coalesced; an unmasked robot costs its mask byte, so k reset robots cost k robots' stores.
__global__ void tick_reset_robots_kernel(int B, const uint8_t* __restrict__ mask, CommandInit P, double* __restrict__ x0, double* __restrict__ gc,
                                         double* __restrict__ tau, double* __restrict__ imu, double* __restrict__ cmd, double* __restrict__ ref,
                                         double* __restrict__ swing, uint32_t* __restrict__ warm, int warm_words, uint8_t* __restrict__ pending) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !mask[b]) return;
  const size_t lb = (size_t)B;
  for (int r = 0; r < 12; ++r) { x0[r * lb + b] = 0.0; tau[r * lb + b] = 0.0; }
  for (int r = 0; r < 4; ++r) gc[r * lb + b] = 0.0;
  if (imu) imu_init_body(b, B, imu);
  command_init_body(b, B, P, cmd, ref, lb);
  swing_init_body(b, B, swing);
  if (warm)
    for (int w = 0; w < warm_words; ++w) warm[(size_t)b * warm_words + w] = 0u;
  if (pending) pending[b] = 1;
}

// stage 6 of the first run after a partial reset, behind the EKF update of every robot: robot b with pending[b] != 0 gets the EKF
// initialisation of ekf_init_kernel instead of the update, and x0 rows 3-5 and 9-11 back at zero, as on the first run of a fresh tick;
// pending[b] is cleared.
__global__ void ekf_init_pending(int B, uint8_t* __restrict__ pending, double* __restrict__ state, const double* __restrict__ foot_pos_rel,
                                 const double* __restrict__ rot, double* __restrict__ x0) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !pending[b]) return;
  ekf_init_body(b, B, state, foot_pos_rel, rot);
  const size_t lb = (size_t)B;
  for (int a = 0; a < 3; ++a) { x0[(3 + a) * lb + b] = 0.0; x0[(9 + a) * lb + b] = 0.0; }
  pending[b] = 0;
}

}  // namespace a1mpc
