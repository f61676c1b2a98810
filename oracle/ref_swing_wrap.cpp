// oracle/ref_swing_wrap.cpp -- TEST INFRASTRUCTURE.  A multi-tick driver around the REFERENCE'S OWN control sources, which
// `make -C oracle -f swing.mk ref` compiles UNMODIFIED from where they lie under /root/reference/src/a1_cpp/src (A1RobotControl.cpp,
// ConvexMpc.cpp, utils/Utils.cpp, ...) against the header stand-ins in oracle/ref_shim/ into oracle/_ref/libref_swing.so -- a library
// of its own, so that its OsqpEigen hook (zeros) never meets the solver installed in oracle/_ref/libref_mpc.so.
//
// What this pins: generate_swing_legs_ctrl (A1RobotControl.cpp:204-287) and the terrain adaptation at the top of compute_grf
// (:334-376, compute_walking_surface :566-582) over many ticks of one controller, filters and all.  tests/golden/make_swing_golden.py
// turns its records into tests/golden/swing_v1.npz so that the GPU box (which has no /root/reference) can check against them.
// Nothing here is product code; nothing under a1-qp-mpc-controller_b200/ may link it.
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

struct CoutMute {  // the reference prints from constructors and from compute_grf
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

// the QP handed to OsqpEigen::Solver::solve() is answered by zeros: only what compute_grf computes before the solve is recorded
int qp_hook_zero(int n, int m, const double*, const double*, const double*, const double*, const double*, int, double* x, double* y) {
  for (int i = 0; i < n; ++i) x[i] = 0.0;
  for (int i = 0; i < m; ++i) y[i] = 0.0;
  return 0;
}

}  // namespace

extern "C" {

// T control ticks of update_plan -> generate_swing_legs_ctrl -> compute_grf (MPC branch) on ONE A1RobotControl / A1CtrlStates pair, so
// that the controller's moving-window filters, last positions and early contacts carry over from tick to tick
// (GazeboA1ROS.cpp:190-191 and the top of compute_grf).  The gait constants and default_foot_pos are A1CtrlStates::reset()'s.
// Per-tick inputs, tick-major: movement_mode [T], lin_vel, lin_vel_d, root_pos [T][3], rot_z, rot [T][9] (row-major), foot_pos_abs [T][12]
// leg-major, foot_force [T][4].  Per-tick outputs: gait_counter [T][4], plan_contacts, contacts [T], foot_pos_target_rel, f_kin
// (foot_forces_kin), foot_pos_cur, foot_pos_recent_contact [T][12], root_euler_d1 and terrain_pitch [T] as the state holds them after
// compute_grf.
int ref_swing_ticks(int T, int use_terrain_adapt, double dt, const double* kp12, const double* kd12, const double* gait_counter_speed4,
                    const int* movement_mode, const double* lin_vel, const double* lin_vel_d, const double* root_pos, const double* rot_z,
                    const double* rot, const double* foot_pos_abs, const double* foot_force, double* gait_counter, uint32_t* plan_contacts,
                    uint32_t* contacts, double* target_rel, double* f_kin, double* foot_pos_cur, double* recent, double* root_euler_d1,
                    double* terrain_pitch) {
  CoutMute mute;
  OsqpEigen::solve_hook() = qp_hook_zero;
  A1RobotControl ctrl;
  A1CtrlStates state;
  state.stance_leg_control_type = 1;
  state.use_terrain_adapt = use_terrain_adapt;
  state.kp_foot = legs(kp12);
  state.kd_foot = legs(kd12);
  for (int i = 0; i < 4; ++i) state.gait_counter_speed(i) = gait_counter_speed4[i];
  state.terrain_pitch_angle = 0;
  for (int t = 0; t < T; ++t) {
    state.movement_mode = movement_mode[t];
    state.root_lin_vel = vec3(lin_vel + 3 * t);
    state.root_lin_vel_d = vec3(lin_vel_d + 3 * t);
    state.root_pos = vec3(root_pos + 3 * t);
    state.root_rot_mat_z = mat3_rowmajor(rot_z + 9 * t);
    state.root_rot_mat = mat3_rowmajor(rot + 9 * t);
    state.foot_pos_abs = legs(foot_pos_abs + 12 * t);
    for (int i = 0; i < 4; ++i) state.foot_force(i) = foot_force[4 * t + i];
    ctrl.update_plan(state, dt);
    ctrl.generate_swing_legs_ctrl(state, dt);
    ctrl.compute_grf(state, dt);
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
    root_euler_d1[t] = state.root_euler_d[1];
    terrain_pitch[t] = state.terrain_pitch_angle;
  }
  return 0;
}

}  // extern "C"
