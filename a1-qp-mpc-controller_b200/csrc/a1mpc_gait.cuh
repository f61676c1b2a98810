// a1mpc_gait.cuh -- per-robot gaits: the kernels of update_plan, the swing legs and the tick's front stage that read each robot's gait
// row instead of the batch-uniform GaitDev / SwingParams and the trot reset (a1mpc_tick_set_gaits, a1mpc_update_plan_gait_batch,
// a1mpc_swing_legs_gait_batch), and the row check.  Include from exactly one translation unit (a1mpc_api.cu), after a1mpc_tick.cuh --
// and from tests/emu (g++, A1MPC_EMU).
//
// A gait row is gait [6][B], batch-major: rows 0-3 the counters a standing robot is reset to (FL FR RL RR), row 4 counter_per_gait (cpg),
// row 5 counter_per_swing (cps).  Each robot loads its cpg and cps once (coalesced); a standing robot also loads its four offsets.
// The swing lasts cpg - cps counts: spline time (g - cps) / (cpg - cps) and the early-contact threshold at the middle of the swing,
// cps + 0.5 (cpg - cps).  With cpg = 2 cps both are the reference's (g - cps) / cps and 1.5 cps to the bit (cpg - cps = cps exactly, and
// cps + 0.5 cps and 1.5 cps are the same exact value rounded once), so a trot row reproduces the plain kernels.
//
// Why these are copies of the plain bodies and not template instantiations of them: giving update_plan_counters, tick_front_b_body and
// the rest a GAIT switch (with the plain path unchanged in every expression) still renumbered the uniform registers of update_plan_kernel
// and tick_front_b, so the plain kernels would no longer be the code the reference-pinned tests certified.  Each function below keeps
// the loop shape of its plain twin (the rolled leg loops of a1mpc_tick.cuh's header note), so that the compiler contracts the same
// products into FMAs and a trot row gives the plain kernels' bits.
#pragma once
#include "a1mpc_tick.cuh"

namespace a1mpc {

struct GaitRow { const double* gait; size_t ld; double cpg, cps; };
__device__ __forceinline__ GaitRow gait_row(const double* __restrict__ gait, size_t ld, int b) {
  return GaitRow{gait, ld, gait[4 * ld + b], gait[5 * ld + b]};
}

// update_plan_counters with the robot's cpg / cps, and its own offsets on standstill (its gait_counter_reset())
__device__ __forceinline__ uint32_t gait_plan_counters(int b, size_t ld, const GaitRow& GR, double* __restrict__ gc, const double* __restrict__ gcs,
                                                       bool walk, double (&c)[4], double (&sp)[4]) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sp[i] = gcs[(size_t)i * ld + b];
    if (!walk) {
      c[i] = GR.gait[(size_t)i * GR.ld + b];
      m |= 1u << i;
    } else {
      c[i] = fmod(gc[(size_t)i * ld + b] + sp[i], GR.cpg);
      if (c[i] <= GR.cps) m |= 1u << i;
    }
    gc[(size_t)i * ld + b] = c[i];
  }
  return m;
}

// update_plan_sched with the robot's cpg / cps; N from G
__device__ __forceinline__ void gait_plan_sched(int b, size_t ld, int N, const GaitRow& GR, bool walk, const double (&c)[4], const double (&sp)[4],
                                                int first, uint32_t* __restrict__ sched) {
  for (int st = first; st < N; ++st) {
    uint32_t ms = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const double ci = walk ? fmod(c[i] + (double)st * sp[i], GR.cpg) : 0.0;
      if (!walk || ci <= GR.cps) ms |= 1u << i;
    }
    sched[(size_t)st * ld + b] = ms;
  }
}

// plan_target_leg with the robot's cps in the Raibert term (cps / sp) * cdt / 2
__device__ __forceinline__ void gait_target_leg(int i, GaitDev G, double cps, double sp, const PlanTargets& T, double (&f)[3]) {
  double dx = T.kf * (T.vr0 - T.vd[0]) + ((cps / sp) * G.cdt) / 2.0 * T.vd[0];
  double dy = T.kf * (T.vr1 - T.vd[1]) + ((cps / sp) * G.cdt) / 2.0 * T.vd[1];
  dx = fmin(fmax(dx, -G.dxl), G.dxl);
  dy = fmin(fmax(dy, -G.dyl), G.dyl);
  f[0] = G.dfp[0 * 4 + i] + dx;
  f[1] = G.dfp[1 * 4 + i] + dy;
  f[2] = G.dfp[2 * 4 + i];
}

// a1mpc_update_plan_gait_batch: update_plan_kernel with each robot's row
__global__ void update_plan_gait_kernel(int B, GaitDev G, const double* __restrict__ gait, double* __restrict__ gc, const double* __restrict__ gcs,
                                        const uint32_t* __restrict__ mode, const double* __restrict__ lv, const double* __restrict__ lvd,
                                        const double* __restrict__ rz, const double* __restrict__ rot, const double* __restrict__ pos,
                                        uint32_t* __restrict__ plan, uint32_t* __restrict__ sched, double* __restrict__ t_rel, double* __restrict__ t_abs,
                                        double* __restrict__ t_world) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  const GaitRow GR = gait_row(gait, ld, b);
  double c[4], sp[4];
  const bool walk = mode[b] != 0;
  const uint32_t m = gait_plan_counters(b, ld, GR, gc, gcs, walk, c, sp);
  plan[b] = m;
  if (sched) gait_plan_sched(b, ld, G.N, GR, walk, c, sp, 0, sched);
  if (t_rel || t_abs || t_world) {
    PlanTargets T;
    plan_targets_setup(b, ld, G, lv, lvd, rz, rot, pos, T);
    for (int i = 0; i < 4; ++i) {
      double f[3];
      gait_target_leg(i, G, GR.cps, sp[i], T, f);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const double fa = T.R[3 * a] * f[0] + T.R[3 * a + 1] * f[1] + T.R[3 * a + 2] * f[2];
        if (t_rel) t_rel[(size_t)(3 * i + a) * ld + b] = f[a];
        if (t_abs) t_abs[(size_t)(3 * i + a) * ld + b] = fa;
        if (t_world) t_world[(size_t)(3 * i + a) * ld + b] = fa + T.p[a];
      }
    }
  }
}

// swing_leg with the robot's cps and cpg (P.cps is not read)
template <class Src>
__device__ __forceinline__ void gait_swing_leg(int i, int b, size_t ld, const SwingParams& P, const GaitRow& GR, double* __restrict__ s,
                                               const double (&R)[9], uint32_t pm, uint32_t& early, uint32_t& cm, const Src& src,
                                               const double* __restrict__ ff, double* __restrict__ fkin, double* __restrict__ cur_out,
                                               double* __restrict__ rc_out) {
  double p[3], cur[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) p[a] = src.p(i, a);
#pragma unroll
  for (int a = 0; a < 3; ++a) cur[a] = R[a] * p[0] + R[3 + a] * p[1] + R[6 + a] * p[2];   // R_z^T p  (:224)
  const double g = src.g(i);
  float t = 0.0f;
  double st[3];
  if (g <= GR.cps) {   // stance: keep refreshing foot_pos_start (:227-232)
#pragma unroll
    for (int a = 0; a < 3; ++a) { st[a] = cur[a]; s[(size_t)(SW_START + 3 * i + a) * ld] = cur[a]; }
  } else {             // swing: spline time in single precision over the swing's cpg - cps counts (:235 with cpg = 2 cps)
    t = (float)(g - GR.cps) / (float)(GR.cpg - GR.cps);
#pragma unroll
    for (int a = 0; a < 3; ++a) st[a] = s[(size_t)(SW_START + 3 * i + a) * ld];
  }
  double fin[3], target[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) fin[a] = src.fin(i, a);
  {
    const double PX[5] = {st[0], st[0], fin[0], fin[0], fin[0]};
    const double PY[5] = {st[1], st[1], fin[1], fin[1], fin[1]};
    const double PZ[5] = {st[2], st[2] + SW_CLEARANCE1, fin[2] + (SW_CLEARANCE2 + 0.5 * 0.0), fin[2], fin[2]};
    const double td = (double)t;
    target[0] = sw_bezier(td, PX); target[1] = sw_bezier(td, PY); target[2] = sw_bezier(td, PZ);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const size_t ir = (size_t)(SW_RLAST + 3 * i + a) * ld, it = (size_t)(SW_TLAST + 3 * i + a) * ld;
    const double vcur = (cur[a] - s[ir]) / P.dt;
    const double vtgt = (target[a] - s[it]) / P.dt;
    s[ir] = cur[a];
    s[it] = target[a];
    const double err = target[a] - cur[a], verr = vtgt - vcur;
    fkin[(size_t)(3 * i + a) * ld + b] = err * P.kp[3 * i + a] + verr * P.kd[3 * i + a];
    if (cur_out) cur_out[(size_t)(3 * i + a) * ld + b] = cur[a];
  }
  // early contact (:259-267) past the middle of the swing (1.5 cps with cpg = 2 cps)
  const bool planned = (pm >> i) & 1u;
  const double mid = GR.cps + 0.5 * (GR.cpg - GR.cps);
  if (g <= mid) early &= ~(1u << i);
  if (!planned && g > mid && ff[(size_t)i * ld + b] > SW_FOOT_FORCE_LOW) early |= 1u << i;
  const bool c = planned || ((early >> i) & 1u);
  if (c) {
    cm |= 1u << i;
#pragma unroll
    for (int a = 0; a < 3; ++a) s[(size_t)(SW_RC + 3 * i + a) * ld] = sw_filter(s, ld, 3 * i + a, p[a]);
  }
  if (rc_out) {
#pragma unroll
    for (int a = 0; a < 3; ++a) rc_out[(size_t)(3 * i + a) * ld + b] = s[(size_t)(SW_RC + 3 * i + a) * ld];
  }
}

// a1mpc_swing_legs_gait_batch: swing_legs_kernel with each robot's row
__global__ void swing_legs_gait_kernel(int B, SwingParams P, const double* __restrict__ gait, double* __restrict__ state, const double* __restrict__ gc,
                                       const uint32_t* __restrict__ plan, const double* __restrict__ rz, const double* __restrict__ fpa,
                                       const double* __restrict__ tgt, const double* __restrict__ ff, double* __restrict__ fkin,
                                       uint32_t* __restrict__ contacts, double* __restrict__ cur_out, double* __restrict__ rc_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  const GaitRow GR = gait_row(gait, ld, b);
  const SwingSrcArrays src{gc, plan, fpa, tgt, ld, b};
  double* s = state + b;
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = rz[(size_t)k * ld + b];
  const uint32_t pm = src.plan();
  uint32_t early = (uint32_t)s[(size_t)SW_EARLY * ld];
  uint32_t cm = 0;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) gait_swing_leg(i, b, ld, P, GR, s, R, pm, early, cm, src, ff, fkin, cur_out, rc_out);
  s[(size_t)SW_EARLY * ld] = (double)early;
  contacts[b] = cm;
}

// tick_front_b_body with each robot's row; sched == nullptr computes no schedule
__device__ __forceinline__ void tick_front_gait_body(int B, const LegParams& LP, const GaitDev& G, const SwingParams& SP, const double* __restrict__ gait,
                                                     const double* __restrict__ joint_pos, const double* __restrict__ joint_vel,
                                                     const double* __restrict__ rot, const double* __restrict__ rot_z, const double* __restrict__ x0,
                                                     const double* __restrict__ lin_vel_d, const uint32_t* __restrict__ mode, double* __restrict__ gc,
                                                     const double* __restrict__ gcs, double* __restrict__ swing_state,
                                                     const double* __restrict__ foot_force, double* __restrict__ fpr, double* __restrict__ jac,
                                                     double* __restrict__ fvr, double* __restrict__ foot, double* __restrict__ fkin,
                                                     uint32_t* __restrict__ contacts, uint32_t* __restrict__ sched) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  double fpa[12];
  leg_kinematics_body(b, ld, joint_pos, joint_vel, rot, LP, fpr, jac, fvr, foot, nullptr, [&](int k, double v) { fpa[k] = v; });
  const GaitRow GR = gait_row(gait, ld, b);
  double c[4], sp[4];
  const bool walk = mode[b] != 0;
  const uint32_t plan = gait_plan_counters(b, ld, GR, gc, gcs, walk, c, sp);
  if (sched) gait_plan_sched(b, ld, G.N, GR, walk, c, sp, 1, sched);
  PlanTargets T;
  plan_targets_setup(b, ld, G, x0 + 9 * ld, lin_vel_d, rot_z, rot, x0 + 3 * ld, T);
  double* s = swing_state + b;
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = rot_z[(size_t)k * ld + b];
  uint32_t early = (uint32_t)s[(size_t)SW_EARLY * ld];
  uint32_t cm = 0;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    double f[3];
    gait_target_leg(i, G, GR.cps, leg_select(sp[0], sp[1], sp[2], sp[3], i), T, f);
    const SwingSrcTick src{gc, plan, fpa, f, ld, b};
    gait_swing_leg(i, b, ld, SP, GR, s, R, plan, early, cm, src, foot_force, fkin, nullptr, nullptr);
  }
  s[(size_t)SW_EARLY * ld] = (double)early;
  contacts[b] = cm;
  if (sched) sched[b] = cm;
}

// the gait twins of tick_front_b and tick_front_sched (a1mpc_tick_set_gaits): gait [6][B], the tick's checked rows
__global__ void tick_front_b_gait(int B, LegParams LP, GaitDev G, SwingParams SP, const double* __restrict__ gait, const double* __restrict__ joint_pos,
                                  const double* __restrict__ joint_vel, const double* __restrict__ rot, const double* __restrict__ rot_z,
                                  const double* __restrict__ x0, const double* __restrict__ lin_vel_d, const uint32_t* __restrict__ mode,
                                  double* __restrict__ gc, const double* __restrict__ gcs, double* __restrict__ swing_state,
                                  const double* __restrict__ foot_force, double* __restrict__ fpr, double* __restrict__ jac, double* __restrict__ fvr,
                                  double* __restrict__ foot, double* __restrict__ fkin, uint32_t* __restrict__ contacts) {
  tick_front_gait_body(B, LP, G, SP, gait, joint_pos, joint_vel, rot, rot_z, x0, lin_vel_d, mode, gc, gcs, swing_state, foot_force, fpr, jac, fvr, foot,
                       fkin, contacts, nullptr);
}

__global__ void tick_front_sched_gait(int B, LegParams LP, GaitDev G, SwingParams SP, const double* __restrict__ gait,
                                      const double* __restrict__ joint_pos, const double* __restrict__ joint_vel, const double* __restrict__ rot,
                                      const double* __restrict__ rot_z, const double* __restrict__ x0, const double* __restrict__ lin_vel_d,
                                      const uint32_t* __restrict__ mode, double* __restrict__ gc, const double* __restrict__ gcs,
                                      double* __restrict__ swing_state, const double* __restrict__ foot_force, double* __restrict__ fpr,
                                      double* __restrict__ jac, double* __restrict__ fvr, double* __restrict__ foot, double* __restrict__ fkin,
                                      uint32_t* __restrict__ contacts, uint32_t* __restrict__ sched) {
  tick_front_gait_body(B, LP, G, SP, gait, joint_pos, joint_vel, rot, rot_z, x0, lin_vel_d, mode, gc, gcs, swing_state, foot_force, fpr, jac, fvr, foot,
                       fkin, contacts, sched);
}

// The rules of a gait row (a1mpc_tick_set_gaits), first broken first: 1 a non-finite entry, 2 not 0 < cps < cpg, 3 an offset outside
// [0, cpg).  bad (one word, preset to all ones by the caller) gets the least (b << 2 | rule) over the robots that break one.
__global__ void gait_check_kernel(int B, const double* __restrict__ gait, unsigned long long* __restrict__ bad) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  double r[6];
  bool finite = true;
#pragma unroll
  for (int k = 0; k < 6; ++k) { r[k] = gait[(size_t)k * ld + b]; finite = finite && isfinite(r[k]); }
  unsigned rule = 0;
  if (!finite) rule = 1;
  else if (!(r[5] > 0.0 && r[5] < r[4])) rule = 2;
  else
    for (int i = 0; i < 4; ++i)
      if (!(r[i] >= 0.0 && r[i] < r[4])) rule = 3;
  if (rule) atomicMin(bad, ((unsigned long long)b << 2) | rule);
}

}  // namespace a1mpc
