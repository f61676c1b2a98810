// oracle/ref_gait_wrap.cpp -- TEST INFRASTRUCTURE.  A multi-tick driver around the REFERENCE'S OWN control sources with a per-robot gait,
// which `make -C oracle -f gait.mk ref` compiles UNMODIFIED from where they lie (A1RobotControl.cpp and the sources it links) against the
// header stand-ins in oracle/ref_shim/ into oracle/_ref/libref_gait.so.
//
// What this pins: update_plan (A1RobotControl.cpp:148-202) and generate_swing_legs_ctrl (:204-287) with a gait row of a1mpc_gait_row
// (offsets, counter_per_gait, counter_per_swing).  The reference fills in gait_counter_reset() only for gait_type 1 (A1CtrlStates.h:322-326),
// so the driver sets gait_type = 0 (the reset then leaves the counters alone), presets gait_counter to the row's offsets on every standstill
// tick, and sets the instance's counter_per_gait / counter_per_swing.  The reference's swing expressions are (g - cps) / cps and 1.5 cps, so
// the rows this pins against the reference's code are those with cpg = 2 cps.  Nothing here is product code.
#include <cstdint>
#include <iostream>
#include <sstream>

#include <Eigen/Dense>
#include "OsqpEigen/OsqpEigen.h"
#include <ros/ros.h>
#include "utils/Utils.h"
#include "A1CtrlStates.h"
#include "ConvexMpc.h"
#include "A1RobotControl.h"

namespace {

struct CoutMute {  // the reference prints from constructors
  std::streambuf* old;
  std::ostringstream sink;
  CoutMute() : old(std::cout.rdbuf(sink.rdbuf())) {}
  ~CoutMute() { std::cout.rdbuf(old); }
};

Eigen::Matrix3d mat3_rowmajor(const double* a) {
  Eigen::Matrix3d m;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) m(i, j) = a[3 * i + j];
  return m;
}
Eigen::Vector3d vec3(const double* a) { return Eigen::Vector3d(a[0], a[1], a[2]); }
Eigen::Matrix<double, 3, NUM_LEG> legs(const double* a) {  // leg-major [3*leg + axis] -> 3 x 4, column = leg
  Eigen::Matrix<double, 3, NUM_LEG> m;
  for (int l = 0; l < NUM_LEG; ++l)
    for (int k = 0; k < 3; ++k) m(k, l) = a[3 * l + k];
  return m;
}
template <class M> void out_legs(const M& m, double* o) {  // 3 x 4 -> leg-major
  for (int l = 0; l < NUM_LEG; ++l)
    for (int k = 0; k < 3; ++k) o[3 * l + k] = m(k, l);
}

}  // namespace

extern "C" {

// T control ticks of update_plan -> generate_swing_legs_ctrl on ONE A1RobotControl / A1CtrlStates pair with the gait row `row`
// (offsets FL FR RL RR, counter_per_gait, counter_per_swing).  Inputs and outputs as ref_swing_ticks of ref_swing_wrap.cpp (no compute_grf,
// so no root_euler_d1 / terrain_pitch).
int ref_gait_ticks(int T, const double* row, double dt, const double* kp12, const double* kd12, const double* gait_counter_speed4,
                   const int* movement_mode, const double* lin_vel, const double* lin_vel_d, const double* root_pos, const double* rot_z,
                   const double* rot, const double* foot_pos_abs, const double* foot_force, double* gait_counter, uint32_t* plan_contacts,
                   uint32_t* contacts, double* target_rel, double* f_kin, double* foot_pos_cur, double* recent) {
  CoutMute mute;
  A1RobotControl ctrl;
  A1CtrlStates state;
  state.stance_leg_control_type = 1;
  state.gait_type = 0;
  state.counter_per_gait = row[4];
  state.counter_per_swing = row[5];
  state.kp_foot = legs(kp12);
  state.kd_foot = legs(kd12);
  for (int i = 0; i < 4; ++i) state.gait_counter_speed(i) = gait_counter_speed4[i];
  for (int t = 0; t < T; ++t) {
    state.movement_mode = movement_mode[t];
    state.root_lin_vel = vec3(lin_vel + 3 * t);
    state.root_lin_vel_d = vec3(lin_vel_d + 3 * t);
    state.root_pos = vec3(root_pos + 3 * t);
    state.root_rot_mat_z = mat3_rowmajor(rot_z + 9 * t);
    state.root_rot_mat = mat3_rowmajor(rot + 9 * t);
    state.foot_pos_abs = legs(foot_pos_abs + 12 * t);
    for (int i = 0; i < 4; ++i) state.foot_force(i) = foot_force[4 * t + i];
    if (!state.movement_mode)
      for (int i = 0; i < 4; ++i) state.gait_counter(i) = row[i];   // the robot's own gait_counter_reset()
    ctrl.update_plan(state, dt);
    ctrl.generate_swing_legs_ctrl(state, dt);
    uint32_t pc = 0, c = 0;
    for (int i = 0; i < 4; ++i) {
      gait_counter[4 * t + i] = state.gait_counter(i);
      pc |= (state.plan_contacts[i] ? 1u : 0u) << i;
      c |= (state.contacts[i] ? 1u : 0u) << i;
    }
    plan_contacts[t] = pc;
    contacts[t] = c;
    out_legs(state.foot_pos_target_rel, target_rel + 12 * t);
    out_legs(state.foot_forces_kin, f_kin + 12 * t);
    out_legs(state.foot_pos_cur, foot_pos_cur + 12 * t);
    out_legs(state.foot_pos_recent_contact, recent + 12 * t);
  }
  return 0;
}

}  // extern "C"
