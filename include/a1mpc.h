/*
 * a1mpc.h -- C ABI of the H100-native batched convex-MPC QP engine.
 *
 * Drop-in boundary for the hot path of ShuoYangRobotics/A1-QP-MPC-Controller:
 *   ConvexMpc            (src/a1_cpp/src/ConvexMpc.h:22-94,  ConvexMpc.cpp:7-260)
 *   A1RobotControl::compute_grf, MPC branch (src/a1_cpp/src/A1RobotControl.cpp:446-562)
 *   A1RobotControl::compute_grf, QP  branch (src/a1_cpp/src/A1RobotControl.cpp:377-445)
 *   OsqpEigen::Solver set-up / solve / getSolution call sites
 *                        (A1RobotControl.cpp:416-439, 522-555; test/test_mpc.cpp:131-151)
 *
 * Plain C, no Eigen / STL / torch types.  Every function returns 0 on success and a negative
 * A1MPC_E* code on failure; a1mpc_last_error() gives the message of the calling thread's last
 * failure.  A handle owns one CUDA device + one stream + scratch; it is NOT thread-safe,
 * distinct handles are independent.  There is no CPU fallback: without a usable CUDA device
 * a1mpc_create() fails with A1MPC_ENODEVICE.
 *
 * Batch layout: every per-QP field is batch-major SoA ("field-major, QP index fastest"):
 * element (field f, QP b) of an array documented as [F][B] lives at  base[f * ld + b]  where
 * ld is the `ld` member of the struct (ld >= B; ld == B for a dense batch).  This is what makes
 * a warp's loads coalesced on the device.
 *
 * Host or device arrays, for every batch entry point (a1mpc_*_batch*): the batch arrays of one call
 * are either ALL host memory or ALL device memory, detected with cudaPointerGetAttributes; a mix is
 * rejected with A1MPC_EINVAL ("all-host or all-device") before anything is enqueued.
 *   host    the call copies its inputs to the device (cudaMemcpy2DAsync where ld > B; pinned memory
 *           from a1mpc_host_alloc makes the copies truly asynchronous DMA, pageable memory works and is
 *           staged by the driver), launches, copies its outputs back and synchronises its stream once:
 *           the call is synchronous.
 *   device  the call only enqueues on the handle's stream (a1mpc_sync) and copies nothing.
 * The batch-uniform parameters that a call reads itself (km_foot, torques_gravity, rho_opt, rho_fix,
 * kp_foot, kd_foot, kd_linear, kp_angular, kd_angular, the command params) are always host memory, and the state buffers (warm,
 * ekf_state, swing_state, imu_state, cmd_state) always device memory; A1MPC_EINVAL otherwise.
 */
#ifndef A1MPC_H_
#define A1MPC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define A1MPC_VERSION 100

/* error codes */
#define A1MPC_OK          0
#define A1MPC_EINVAL     -1   /* bad argument / unsupported configuration            */
#define A1MPC_ENODEVICE  -2   /* no usable CUDA device (there is no CPU fallback)    */
#define A1MPC_ECUDA      -3   /* CUDA runtime error, see a1mpc_last_error()          */
#define A1MPC_ENOMEM     -4
#define A1MPC_ENCCL      -5   /* NCCL not loadable / NCCL error                      */

/* per-QP status written by the solve kernels */
#define A1MPC_STATUS_OPTIMAL     0  /* KKT certificate verified in-kernel (exact active set)  */
#define A1MPC_STATUS_IPM_ONLY    1  /* interior-point iterate returned, finisher not verified */
#define A1MPC_STATUS_MAXITER     2  /* iteration cap hit before the IPM tolerance             */
#define A1MPC_STATUS_NUMERICAL   3  /* non-positive pivot / NaN in the inputs                 */
#define A1MPC_STATUS_NO_CONTACT  4  /* no stance foot: all forces are zero by the constraints */

#define A1MPC_MAX_HORIZON 20

typedef struct a1mpc_handle a1mpc_handle;

/* Batch-uniform configuration; mirrors the constants of the reference.
 *   horizon          PLAN_HORIZON                      (A1Params.h:26)            10 | 20
 *   dt               mpc_dt                            (A1RobotControl.cpp:462)
 *   mu,fz_min,fz_max friction pyramid and fz bounds    (ConvexMpc.cpp:8, 223-224)
 *   mass, inertia    robot_mass, a1_trunk_inertia      (A1CtrlStates.h:40-43), row-major
 *   q[13], r[12]     q_weights, r_weights (un-doubled; the engine applies the factor 2 of
 *                    ConvexMpc.cpp:20,41)
 *   max_iter, tol    solver controls; 0 selects the defaults (40, 1e-9 switch-over mu)
 *   precision        64: every array of the boundary is fp64 (the reference's arithmetic type).
 *                    32: BASELINE config 3's "fp32" -- the floating-point arrays of the HOT-PATH boundary (a1mpc_solve_batch,
 *                        a1mpc_solve_batch_warm, a1mpc_solve_batch_ext: x0, rot, foot, ref, normals in; f_body, u_full out) hold
 *                        float instead of double, 224 instead of 440 bytes per QP; they are declared `double*` below and
 *                        reinterpreted.  The arithmetic in between stays fp64 with the in-kernel KKT certificate: the reduced
 *                        systems have condition numbers of 1e5 (N=10) .. 1e6 (N=20), an fp32 factorisation cannot certify
 *                        1e-4 N, and the only fp32-input tensor-core MMA (tf32, 10-bit mantissa) breaks down on 85 % of the
 *                        QPs.  Accuracy contract: the returned forces are the exact optimum of the QP
 *                        posed by the fp32-rounded inputs, rounded to fp32 -- |f - f*(rounded inputs)| <= 1e-4 N + 1 fp32 ulp.
 *                        The parity / neighbouring entry points (build_qp, qp_mats, solve_dense, grf_qp, stance_qp, torques, plan,
 *                        kinematics, EKF) are fp64 whatever this field says.
 */
typedef struct a1mpc_config {
  int    horizon;
  int    precision;      /* 64 | 32 (fp32 arrays at the hot-path boundary, see above)  */
  double dt;
  double mu, fz_min, fz_max;
  double mass;
  double inertia[9];
  double q[13];
  double r[12];
  int    max_iter;
  double tol;
} a1mpc_config;

/* Fills cfg with the reference launch defaults (config/gazebo_a1_mpc.yaml:6-72,
 * a1_ctrl.launch:2-3): N=10, dt=0.0025, mu=0.3, fz in [0,180], mass 12, gazebo weights. */
void a1mpc_default_config(a1mpc_config* cfg);

/* Inputs of A1RobotControl::compute_grf's MPC branch, i.e. the A1CtrlStates fields it reads
 * (A1RobotControl.cpp:452-488, 498-503; A1CtrlStates.h:347-413).
 *   x0     [12][B]  root_euler(3), root_pos(3), root_ang_vel(3), root_lin_vel(3)  (world)
 *   rot     [9][B]   root_rot_mat, row-major
 *   foot    [12][B]  foot_pos_abs, leg-major: FL(x,y,z), FR, RL, RR  (A1CtrlStates.h:399)
 *   ref     [9][B]   root_euler_d[0], root_euler_d[1], root_ang_vel_d(3), root_lin_vel_d(3, body),
 *                    root_pos_d[2]
 *   contact [B]      bit i set = state.contacts[i]   (leg order FL,FR,RL,RR)
 */
typedef struct a1mpc_inputs {
  const double*   x0;
  const double*   rot;
  const double*   foot;
  const double*   ref;
  const uint32_t* contact;
  size_t          ld;
} a1mpc_inputs;

/* Outputs.  f_body is what compute_grf returns (A1RobotControl.cpp:555-563): R^T * u[3i:3i+3],
 * first horizon step, leg-major.  status is mandatory; iters and u_full may be NULL.
 *   f_body [12][B]   status [B]   iters [B] (IPM iterations + 100*finisher rounds)
 *   u_full [12*N][B] world-frame solution over the whole horizon (OsqpEigen getSolution()) */
typedef struct a1mpc_outputs {
  double*  f_body;
  int32_t* status;
  int32_t* iters;
  double*  u_full;
  size_t   ld;
} a1mpc_outputs;

/* ---- life cycle --------------------------------------------------------------------------- */
int  a1mpc_create(a1mpc_handle** out, const a1mpc_config* cfg, int device);
int  a1mpc_destroy(a1mpc_handle* h);
const char* a1mpc_last_error(void);
int  a1mpc_device_count(void);

/* ---- the hot path: replaces compute_grf's MPC branch for B robots -------------------------- */
/* One call = build (linearise, condense, Hessian, gradient) + QP solve + force extraction for
 * every QP of the batch.  Host or device arrays as stated at the top of this file. */
int  a1mpc_solve_batch(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_outputs* out);

/* ---- device-resident warm start across control ticks (SURVEY 8f.3) --------------------------------------------------
 * The reference keeps ONE OsqpEigen::Solver alive and warm-starts every tick from the previous solution
 * (A1RobotControl.h:67, A1RobotControl.cpp:522-538).  Here the state that is worth keeping is the optimal ACTIVE FACE of
 * every robot: a1mpc_solve_batch_warm first runs the exact active-face finisher on the faces stored in `warm` by the
 * previous call (a few reduced factorisations, no interior-point iteration when they still verify -- KKT-certified like
 * every OPTIMAL result) and falls back to the cold path per robot otherwise; it then stores the new faces.  Results are
 * the same optimum either way (the QP is strictly convex).
 *   warm   DEVICE buffer of a1mpc_warm_bytes(h, B) bytes (a1mpc_device_alloc), owned by the caller, one slot per batch
 *          index b; a1mpc_warm_reset (or zero bytes) = no guess.  A robot whose stance feet changed starts cold.
 *   shift  how many horizon steps the stored faces move towards "now" (0: the problem is re-posed relative to the
 *          current state every tick, as compute_grf does; 1: references fixed in absolute time).
 * in / out as in a1mpc_solve_batch (host or device).  Horizon 10 only in this round (A1MPC_EINVAL otherwise). */
size_t a1mpc_warm_bytes(const a1mpc_handle* h, int B);
int  a1mpc_warm_reset(a1mpc_handle* h, void* warm, int B);
int  a1mpc_solve_batch_warm(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_outputs* out, void* warm, int shift);

/* ---- BASELINE config 4: an EXTENSION beyond the reference (which keeps one contact pattern over the horizon,
 * ConvexMpc.cpp:226-245, and world-z friction pyramids) ------------------------------------------------ */
/*   contact_sched [N][B]  contact mask of every horizon step (batch-major, ld of `in`), or NULL = in->contact everywhere
 *   normals       [12][B] terrain normal per foot (world frame, normalised by the engine), or NULL = world z.
 * With normals the friction pyramid and the fz bounds act in each foot's terrain frame; the returned forces are
 * world/body-frame as in a1mpc_solve_batch.  Restrictions: normals need r[3i] == r[3i+1] == r[3i+2] per foot (a rotated
 * diagonal R would not be diagonal), normal z-components must be positive. */
typedef struct a1mpc_inputs_ext {
  const uint32_t* contact_sched;
  const double*   normals;
} a1mpc_inputs_ext;
int  a1mpc_solve_batch_ext(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_inputs_ext* ext, const a1mpc_outputs* out);

/* ---- warm start of the scheduled call: a1mpc_solve_batch_ext + the device-resident warm start above -------------------
 * Same contract as a1mpc_solve_batch_ext (host or device arrays, precision 32, isotropic r with normals) plus `warm` and
 * `shift` as in a1mpc_solve_batch_warm (same buffer: a1mpc_warm_bytes / a1mpc_warm_reset).  The slot keeps the verified face of
 * every (horizon step, leg) together with the schedule it was solved for; the guess for foot-step (st, leg) in contact now is
 * the stored face of (st + shift, leg) (step N-1 past the end) if that foot-step was in contact then, and the free face if it
 * was not.  A schedule produced by a1mpc_update_plan_batch moves by one step per control tick: shift = 1.  A robot whose
 * guess does not verify takes the cold path inside the same launch; OPTIMAL is KKT-certified either way.  Slots written by
 * a1mpc_solve_batch_warm are "no guess" here and the reverse; robots that end NUMERICAL or have no contact store no guess.
 * ext NULL (or both fields NULL) = a1mpc_solve_batch_warm.  A1MPC_EINVAL: horizon 20, shift outside [0, N], `warm` not device
 * memory. */
int  a1mpc_solve_batch_ext_warm(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_inputs_ext* ext, const a1mpc_outputs* out,
                                void* warm, int shift);

/* ---- ConvexMpc members, for parity with the reference class (ConvexMpc.h:87-93) ----------- */
/* Dense QP data exactly as ConvexMpc::calculate_qp_mats leaves it after compute_grf drove it
 * (constant B_d over the horizon, A1RobotControl.cpp:498-514).  QP-major outputs:
 *   H [B][12N][12N] row-major (hessian, densified), g [B][12N] (gradient),
 *   lb, ub [B][20N] (ConvexMpc.cpp:223-245; +-1e30 = OsqpEigen::INFTY).  Any may be NULL. */
int  a1mpc_build_qp_batch(a1mpc_handle* h, int B, const a1mpc_inputs* in,
                          double* H, double* g, double* lb, double* ub);

/* ConvexMpc::calculate_qp_mats for caller-supplied discrete models (the public API allows a
 * different B_d per step: test/test_mpc.cpp:106-122).  QP-major inputs:
 *   A_d [B][13][13] row-major, B_d_list [B][13N][12] row-major (B_mat_d_list),
 *   x0 [B][13] (mpc_states), x_d [B][13N] (mpc_states_d);  outputs as above. */
int  a1mpc_qp_mats_batch(a1mpc_handle* h, int B, const double* A_d, const double* B_d_list,
                         const double* x0, const double* x_d, double* H, double* g);
/* The same call with the intermediate public members of ConvexMpc as well (ConvexMpc.h:77-78, ConvexMpc.cpp:181-202):
 *   A_qp [B][13N][13] (rows 13i.. = A_d^(i+1)),  B_qp [B][13N][12N] (block (i,j) = A_d^(i-j) B_d[j], j <= i, zero above).
 * Any output may be NULL (at least one must not be). */
int  a1mpc_qp_rollout_batch(a1mpc_handle* h, int B, const double* A_d, const double* B_d_list,
                            const double* x0, const double* x_d, double* A_qp, double* B_qp, double* H, double* g);

/* OsqpEigen::Solver replacement for the MPC QP (A1RobotControl.cpp:522-555):
 *   min 1/2 u'Hu + g'u  s.t. the friction pyramid of ConvexMpc.cpp:46-58 with the contact
 *   pattern `contact` (constant over the horizon).  H [B][12N][12N], g [B][12N] QP-major,
 *   u [B][12N] out (getSolution()), status [B].
 *   Only the upper triangle of H is read (as OSQP takes it), and only the rows and columns of the
 *   stance feet: the strict lower triangle and the swing rows, columns and gradient entries may
 *   hold anything.  A stance entry of H or g that is NaN, Inf or of magnitude >= 1e300, or a stance
 *   diagonal entry <= 0, gives NUMERICAL with u all zero.  No stance foot: NO_CONTACT, u zero.
 *   N = 10 serves every stance count; N = 20 one or two feet, while three or four end NUMERICAL
 *   with u zero (their dense factor does not fit in shared memory). */
int  a1mpc_solve_dense_batch(a1mpc_handle* h, int B, const double* H, const double* g,
                             const uint32_t* contact, double* u, int32_t* status);

/* ---- compute_grf's QP branch (stance_leg_control_type == 0), A1RobotControl.cpp:377-445 ---- */
/* 12-variable instantaneous GRF QP, batched.  All arrays QP-major:
 *   root_acc [B][6]  desired wrench (A1RobotControl.cpp:379-391, caller-computed PD + gravity; a1mpc_stance_qp_batch below computes it)
 *   rot_z [B][9], rot [B][9]  root_rot_mat_z, root_rot_mat (row-major); foot [B][12] leg-major
 *   contact [B];  f_body [B][12] out;  status [B] out.
 * Constants Q=diag(1,1,1,400,400,100), R=1e-3, mu=0.7, F in [0,180] (A1RobotControl.cpp:11-15). */
int  a1mpc_grf_qp_batch(a1mpc_handle* h, int B, const double* root_acc, const double* rot_z,
                        const double* rot, const double* foot, const uint32_t* contact,
                        double* f_body, int32_t* status);

/* ---- compute_grf's QP branch from the controller state (stance_leg_control_type == 0, A1RobotControl.cpp:325-333, 377-445), batched ----
 * The PD law in front of the QP (the euler-error wrap of :327-332 with the literal 3.1415926, :379-391 with robot_mass = the
 * handle's cfg.mass and gravity 9.8), then the QP of a1mpc_grf_qp_batch (same constants, same solver, same certificate).  Batch-major
 * SoA with leading dimension ld >= B, so that the x0, rot and foot arrays of an a1mpc_inputs can be passed as they are; host or device:
 *   x0 [12][B]  root_euler(3), root_pos(3), root_ang_vel(3), root_lin_vel(3) (the a1mpc_inputs.x0 layout)
 *   rot [9][B], rot_z [9][B]  root_rot_mat, root_rot_mat_z (row-major);  foot [12][B] foot_pos_abs, leg-major;  contact [B]
 *   des [12][B]  root_euler_d(3), root_pos_d(3), root_lin_vel_d(3, body frame), root_ang_vel_d(3)
 *   kp_linear [3][B]  per robot: the reference zeroes its x and y while a walking robot has a velocity command (GazeboA1ROS.cpp:164-188)
 *   kd_linear[3], kp_angular[3], kd_angular[3]: batch-uniform HOST arrays, like km_foot
 *   out: f_body [12][B] foot_forces_grf (body frame, the f_grf input of a1mpc_joint_torques_batch); status [B];
 *        root_acc [6][B] the desired wrench the QP was posed with (may be NULL).
 * A robot without a stance foot gets A1MPC_STATUS_NO_CONTACT, one whose QP data are not finite A1MPC_STATUS_NUMERICAL; both zero forces.
 * fp64 whatever cfg.precision says. */
int  a1mpc_stance_qp_batch(a1mpc_handle* h, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                           const uint32_t* contact, const double* des, const double* kp_linear, const double* kd_linear,
                           const double* kp_angular, const double* kd_angular, double* f_body, int32_t* status, double* root_acc);
/* a1mpc_stance_qp_batch with each stance foot's friction pyramid on the walking surface rather than world z.  normals [12][ld]: per foot
 * (leg-major, x y z), world frame, host or device like the other batch arrays; the engine normalises them as a1mpc_solve_batch_ext does.
 * Each stance foot's force is solved in the foot's terrain frame T(n) (the rotation about z x n that takes world z to n, the frame of the
 * a1mpc_solve_batch_ext pyramids, so a foot gets the same pyramid in QP and MPC mode): |t_x|, |t_y| <= 0.7 f_n and 0 <= f_n <= 180 act on
 * T(n)^T f_world.  The QP is the same in the world forces, H = R I + M^T Q M, g = -M^T Q root_acc.  f_body is R^T T u_local.
 * A stance foot whose normal is not finite, or has n_z <= 0 after normalisation, makes the robot A1MPC_STATUS_NUMERICAL with zero forces;
 * a swing foot's normal is not read.  All-e_z normals give exactly what a1mpc_stance_qp_batch gives; normals == NULL is that call.
 * fp64 whatever cfg.precision says. */
int  a1mpc_stance_qp_batch_ext(a1mpc_handle* h, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                               const uint32_t* contact, const double* des, const double* kp_linear, const double* kd_linear,
                               const double* kp_angular, const double* kd_angular, const double* normals, double* f_body, int32_t* status,
                               double* root_acc);

/* ---- the step right after the path (SURVEY 8f.1): A1RobotControl::compute_joint_torques ------------- */
/* A1RobotControl.cpp:289-319, batched, batch-major SoA like a1mpc_solve_batch (ld = B), host or device pointers:
 *   f_grf   [12][B]  foot_forces_grf, leg-major (the f_body output of a1mpc_solve_batch can be passed as is)
 *   f_kin   [12][B]  foot_forces_kin, leg-major (swing-leg PD force, A1RobotControl.cpp:286)
 *   jac     [36][B]  the four 3x3 diagonal blocks of j_foot, leg-major then row-major (A1CtrlStates.h:409)
 *   contact [B]      bit i = contacts[i]
 *   km_foot[3], torques_gravity[12]: batch-uniform (A1CtrlStates.h:122,129), host arrays
 *   tau     [12][B]  in/out: stance legs  J^T (-f_grf),  swing legs  J^-1 (km_foot .* f_kin)  (partial-pivot LU),
 *                    + torques_gravity; an entry whose result is NaN keeps its previous value (:314-317). */
int  a1mpc_joint_torques_batch(a1mpc_handle* h, int B, const double* f_grf, const double* f_kin, const double* jac,
                               const uint32_t* contact, const double* km_foot, const double* torques_gravity, double* tau);

/* ---- upstream producers of the path's inputs (SURVEY 8f.4) ------------------------------------------------------ */
/* Leg forward kinematics and Jacobian: A1Kinematics::fk / jac (legKinematics/A1Kinematics.cpp:7-18; bodies :39-131) with the
 * per-tick derived quantities of GazeboA1ROS.cpp:264-279, batched.  Batch-major SoA (ld = B), host or device pointers:
 *   joint_pos [12][B] leg-major (FL, FR, RL, RR) x (hip, thigh, calf); joint_vel [12][B] (NULL: no velocities)
 *   rot [9][B] root_rot_mat row-major (NULL: no *_abs outputs)
 *   rho_opt [12] = 4 legs x (cx, cy, cz) contact offset; rho_fix [20] = 4 legs x (leg_offset_x, leg_offset_y, motor_offset,
 *   upper_leg_length, lower_leg_length) (GazeboA1ROS.cpp:76-97): HOST arrays, batch-uniform
 *   out (any may be NULL): foot_pos_rel [12][B]; jac [36][B] = the four 3x3 blocks of j_foot, leg-major then row-major (the
 *   layout a1mpc_joint_torques_batch takes); foot_vel_rel [12][B] = J dq; foot_pos_abs [12][B] = R foot_pos_rel (the `foot`
 *   input of a1mpc_solve_batch); foot_vel_abs [12][B]. */
int  a1mpc_leg_kinematics_batch(a1mpc_handle* h, int B, const double* joint_pos, const double* joint_vel, const double* rot,
                                const double* rho_opt, const double* rho_fix, double* foot_pos_rel, double* jac, double* foot_vel_rel,
                                double* foot_pos_abs, double* foot_vel_abs);

/* A1BasicEKF (A1BasicEKF.cpp), batched: 18 states (position, velocity, four foot positions), 28 measurements, orientation
 * taken from the IMU.  The filter state lives on the device: a1mpc_ekf_bytes(B) bytes (a1mpc_device_alloc), per robot 342
 * doubles = x[18], P[18][18] row-major.
 *   a1mpc_ekf_init_batch    A1BasicEKF::init_state (:56-68): P = 3 I, x = (0, 0, 0.09, 0, 0, 0, R fk_i + pos)
 *   a1mpc_ekf_update_batch  A1BasicEKF::update_estimation (:70-164) with the constructor's C, Q, R (:7-53; noise constants of
 *                           A1BasicEKF.h:16-21): contact estimate from movement_mode / foot_force, process update, measurement,
 *                           S = C Pbar C' + R, x and P update, position-drift cut (:144-148)
 *   batch-major SoA inputs (ld = B), host or device: movement_mode [B], imu_acc [3][B], imu_ang_vel [3][B], rot [9][B],
 *   foot_pos_rel [12][B], foot_vel_rel [12][B], foot_force [4][B]
 *   out (any may be NULL): root_pos [3][B] (= estimated_root_pos), root_lin_vel [3][B], estimated_contacts [B] (bit i = leg i),
 *   status [B]: 0, or A1MPC_STATUS_NUMERICAL when S is not positive definite / not finite (that robot's state is untouched).
 *   Non-finite input: a NaN or Inf in imu_acc, imu_ang_vel, rot, foot_pos_rel or foot_vel_rel, or a NaN foot_force in walking
 *   mode (the contact estimate min(max(force / 100, 0), 1) keeps the NaN, as the reference's std::min / std::max do), makes the
 *   robot NUMERICAL: its state is untouched, root_pos / root_lin_vel are that state's, and a NaN force's contact bit is 1 (the
 *   reference's ec < 0.5 test is false for NaN).  +-Inf force in walking mode clamps to contact 1 / 0, and standstill ignores the
 *   force: neither is NUMERICAL. */
size_t a1mpc_ekf_bytes(int B);
int  a1mpc_ekf_init_batch(a1mpc_handle* h, int B, void* ekf_state, const double* foot_pos_rel, const double* rot);
int  a1mpc_ekf_update_batch(a1mpc_handle* h, int B, void* ekf_state, double dt, int assume_flat_ground, const uint32_t* movement_mode,
                            const double* imu_acc, const double* imu_ang_vel, const double* rot, const double* foot_pos_rel,
                            const double* foot_vel_rel, const double* foot_force, double* root_pos, double* root_lin_vel,
                            uint32_t* estimated_contacts, int32_t* status);

/* ---- the step right before the path (SURVEY 8f.2): A1RobotControl::update_plan ------------------------ */
/* Gait counters -> planned contacts, and the Raibert foothold targets (A1RobotControl.cpp:148-202), batched; plus what the
 * reference does not do: the planned contact mask of every horizon step (it freezes the current pattern,
 * ConvexMpc.cpp:226-245), in the [N][B] layout a1mpc_solve_batch_ext takes.  Batch-major SoA (ld = B), host or device:
 *   gait_counter [4][B] in/out; gait_counter_speed [4][B]; movement_mode [B] (0 standstill: all feet planned in contact and
 *   the counters reset to the trot offsets 0,120,120,0 -- A1CtrlStates.h:322-326);
 *   lin_vel [3][B] root_lin_vel (world); lin_vel_d [3][B] root_lin_vel_d; rot_z [9][B], rot [9][B], root_pos [3][B];
 *   out: plan_contacts [B]; contact_sched [N][B] (step i = i plan ticks ahead; may be NULL);
 *        foot_pos_target_rel / _abs / _world [12][B] leg-major (any may be NULL). */
typedef struct a1mpc_gait_params {
  double counter_per_gait;      /* 240  (A1CtrlStates.h:23)  */
  double counter_per_swing;     /* 120  (A1CtrlStates.h:24)  */
  double control_dt;            /* MAIN_UPDATE_FREQUENCY / 1000 (A1CtrlStates.h:332) */
  double default_foot_pos[12];  /* 3 x NUM_LEG row-major (A1CtrlStates.h:45-47) */
  double foot_delta_x_limit, foot_delta_y_limit;   /* A1Params.h:44-45 */
  int    horizon;               /* steps of contact_sched */
} a1mpc_gait_params;
int  a1mpc_update_plan_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, double* gait_counter, const double* gait_counter_speed,
                             const uint32_t* movement_mode, const double* lin_vel, const double* lin_vel_d, const double* rot_z,
                             const double* rot, const double* root_pos, uint32_t* plan_contacts, uint32_t* contact_sched,
                             double* foot_pos_target_rel, double* foot_pos_target_abs, double* foot_pos_target_world);
/* Per-robot gaits.  A gait row is six numbers per robot, gait [6][B] batch-major (host or device, like the other arrays):
 *   rows 0-3  the counters a standing robot is reset to, FL FR RL RR (the robot's own gait_counter_reset(), A1CtrlStates.h:322-326)
 *   row 4     counter_per_gait (cpg)
 *   row 5     counter_per_swing (cps: a leg is planned in contact while its counter is <= cps, so cps is the stance length)
 * A valid row is finite, with 0 < cps < cpg and every offset in [0, cpg).  The swing lasts cpg - cps counts: the swing spline time is
 * float(gc - cps) / float(cpg - cps) and the early-contact threshold the middle of the swing, cps + 0.5 (cpg - cps); the foothold's
 * (cps / speed) * control_dt / 2 and the schedule's fmod(c + st * speed, cpg) <= cps take the robot's own cps and cpg.  With cpg = 2 cps
 * (the default 240 / 120) every one of them is the reference's expression to the bit.
 * a1mpc_gait_row fills one row: A1MPC_GAIT_TROT is the reference's gait_type 1, the only one it fills in.  At equal leg speeds the pace
 * swings the lateral pairs together, the bound the front and the rear pair, the pronk all four feet (a flight phase with no foot down);
 * the walk is a lateral-sequence walk (RL, FL, RR, FR a quarter cycle apart, cps = 3/4 cpg) with at most one foot in swing.
 * A1MPC_EINVAL for an unknown type or a NULL row. */
#define A1MPC_GAIT_TROT  1   /* offsets 0 120 120 0,   cpg 240, cps 120 */
#define A1MPC_GAIT_PACE  2   /* offsets 0 120 0 120,   cpg 240, cps 120 */
#define A1MPC_GAIT_BOUND 3   /* offsets 0 0 120 120,   cpg 240, cps 120 */
#define A1MPC_GAIT_PRONK 4   /* offsets 0 0 0 0,       cpg 240, cps 120 */
#define A1MPC_GAIT_WALK  5   /* offsets 120 0 180 60,  cpg 240, cps 180 */
int  a1mpc_gait_row(int gait_type, double row[6]);
/* a1mpc_update_plan_batch with each robot's gait row: gait [6][B] replaces gp's counter_per_gait and counter_per_swing and the trot
 * reset; gp gives the rest.  The rows are not checked here (a1mpc_tick_set_gaits checks them). */
int  a1mpc_update_plan_gait_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* gait, double* gait_counter,
                                  const double* gait_counter_speed, const uint32_t* movement_mode, const double* lin_vel, const double* lin_vel_d,
                                  const double* rot_z, const double* rot, const double* root_pos, uint32_t* plan_contacts, uint32_t* contact_sched,
                                  double* foot_pos_target_rel, double* foot_pos_target_abs, double* foot_pos_target_world);

/* ---- the stages between update_plan and the path: A1RobotControl::generate_swing_legs_ctrl and compute_grf's terrain adaptation ----
 * generate_swing_legs_ctrl (A1RobotControl.cpp:204-287) produces the `contact` of a1mpc_solve_batch* and the f_kin / contact of
 * a1mpc_joint_torques_batch; the front of compute_grf (:334-376, compute_walking_surface :566-582) poses root_euler_d[1] on a slope.
 * The controller state they keep lives on the device: a1mpc_swing_bytes(B) bytes (a1mpc_device_alloc), per robot the fields
 * foot_pos_start, foot_pos_rel_last_time, foot_pos_target_last_time, foot_pos_recent_contact, early_contacts and the thirteen
 * moving-window filters (recent_contact_{x,y,z}_filter[4] of 60 samples, terrain_angle_filter of 100).  The layout is opaque and
 * batch-major, so a buffer is bound to the B it was initialised for: pass the same B to every call on it.
 *   a1mpc_swing_init_batch     A1CtrlStates::reset() values of those fields (A1CtrlStates.h:83-100) and fresh filters
 *                              (A1RobotControl.cpp:52-57): zero positions, no early contact, empty windows
 *   a1mpc_swing_legs_batch     one generate_swing_legs_ctrl tick: foot_pos_cur = R_z^T foot_pos_abs; stance legs (gait_counter <=
 *                              counter_per_swing) refresh foot_pos_start, swing legs follow the degree-4 Bezier from foot_pos_start to
 *                              foot_pos_target_rel with spline time float(gc - cps) / float(cps) and the clearances 0.0f / 0.4f of
 *                              A1Params.h:41-42; finite-difference velocities over dt; f_kin = kp .* pos_error + kd .* vel_error;
 *                              early contact (sticky until gc <= 1.5 cps) when a swing foot past 1.5 cps feels more than FOOT_FORCE_LOW
 *                              = 30 N; contacts = plan | early; on contact ticks the leg's recent-contact filters take foot_pos_abs.
 *                              gp: counter_per_swing only.  kp_foot[12], kd_foot[12] (leg-major: FL(x,y,z), FR, RL, RR): batch-uniform
 *                              HOST arrays, like km_foot.  Batch-major SoA (ld = B), host or device: gait_counter [4][B] (after
 *                              a1mpc_update_plan_batch), plan_contacts [B], rot_z [9][B] root_rot_mat_z, foot_pos_abs [12][B],
 *                              foot_pos_target_rel [12][B], foot_force [4][B]; out: f_kin [12][B] (foot_forces_kin), contacts [B];
 *                              foot_pos_cur, foot_pos_recent_contact [12][B] (may be NULL).
 *   a1mpc_terrain_pitch_batch  least-squares plane through the four recent-contact points (pseudo-inverse with the reference's
 *                              cutoff eps * 3 * sigma_max), dihedral angle to flat ground, averaged by the 100-sample filter only while
 *                              root_pos z > 0.1 (0 otherwise), clipped to +-0.5; the sign is - when the front feet stand more than
 *                              0.05 m above the rear ones.  root_pos [3][B]; ref [9][B] with leading dimension ref_ld >= B, an
 *                              a1mpc_inputs.ref array: only row 1 (root_euler_d[1]) is written, and only when use_terrain_adapt (ref may
 *                              be NULL otherwise); terrain_pitch [B] out (terrain_pitch_angle, may be NULL).
 *   a1mpc_terrain_normals_batch  a1mpc_terrain_pitch_batch (the same filter update, ref row 1 and terrain_pitch) that also writes
 *                              normals [12][B] (mandatory): the walking surface's unit normal in the world frame, the same for all four
 *                              feet, as the per-foot normals of a1mpc_solve_batch_ext take it.  It is the fitted plane's own normal
 *                              (-a1, -a2, 1) / |.| (z = a0 + a1 x + a2 y in the frame of foot_pos_recent_contact, which has world
 *                              axes), its tilt clipped to 0.5 rad about the same horizontal axis, and e_z while root_pos z <= 0.1;
 *                              so n_z >= cos 0.5 > 0.  It advances the same filter: a chain calls one of the two, never both.
 *   a1mpc_surface_normals_batch  the normals of a1mpc_terrain_normals_batch, bit for bit, without its terrain stage: swing_state (device
 *                              memory) is only read, no filter advances and no ref is written.  The reference adapts to terrain only in
 *                              MPC mode, so this is the walking surface of a QP-mode chain (a1mpc_tick_set_stance_terrain's ESTIMATED
 *                              source, staged).  root_pos [3][B] in, normals [12][B] out, host or device.
 */
size_t a1mpc_swing_bytes(int B);
int  a1mpc_swing_init_batch(a1mpc_handle* h, int B, void* swing_state);
int  a1mpc_swing_legs_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* kp_foot, const double* kd_foot, void* swing_state,
                            double dt, const double* gait_counter, const uint32_t* plan_contacts, const double* rot_z, const double* foot_pos_abs,
                            const double* foot_pos_target_rel, const double* foot_force, double* f_kin, uint32_t* contacts, double* foot_pos_cur,
                            double* foot_pos_recent_contact);
/* a1mpc_swing_legs_batch with each robot's gait row gait [6][B] (a1mpc_update_plan_gait_batch): cps and cpg come from the row (gp's
 * counter_per_swing is not read), with the spline time and early-contact threshold of the gait rows above. */
int  a1mpc_swing_legs_gait_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* gait, const double* kp_foot, const double* kd_foot,
                                 void* swing_state, double dt, const double* gait_counter, const uint32_t* plan_contacts, const double* rot_z,
                                 const double* foot_pos_abs, const double* foot_pos_target_rel, const double* foot_force, double* f_kin,
                                 uint32_t* contacts, double* foot_pos_cur, double* foot_pos_recent_contact);
int  a1mpc_terrain_pitch_batch(a1mpc_handle* h, int B, void* swing_state, int use_terrain_adapt, const double* root_pos, double* ref, size_t ref_ld,
                               double* terrain_pitch);
int  a1mpc_terrain_normals_batch(a1mpc_handle* h, int B, void* swing_state, int use_terrain_adapt, const double* root_pos, double* ref,
                                 size_t ref_ld, double* terrain_pitch, double* normals);
int  a1mpc_surface_normals_batch(a1mpc_handle* h, int B, const void* swing_state, const double* root_pos, double* normals);

/* ---- the first two stages of a control tick: the adapters' orientation and command stages ---------------------------------
 * Together with the stages above they let a whole tick run from raw sensor arrays on device pointers.  One thread per robot;
 * batch-major SoA, host or device arrays; the state buffers are device memory (a1mpc_device_alloc), opaque and batch-major, so a
 * buffer is bound to the B it was initialised for.
 *
 * a1mpc_orientation_batch: the IMU and pose callbacks (GazeboA1ROS.cpp:235-299, HardwareA1ROS.cpp:262-276, IsaacA1ROS.cpp:183-241).
 *   quat [4][B] (w, x, y, z: the Quaterniond(w, x, y, z) argument order), gyro [3][B], acc [3][B] (may be NULL): the raw readings.
 *   imu_state  a1mpc_imu_bytes(B) bytes, a1mpc_imu_init_batch: the six MovingWindowFilter(5) of acc and gyro (GazeboA1ROS.cpp:100-105,
 *              IsaacA1ROS.cpp:62-67; utils/filter.hpp), through which each call first passes its sample.  NULL = unfiltered, as on
 *              the hardware adapter (HardwareA1ROS.cpp:273-274).
 *   outputs, each may be NULL:
 *     rot [9][ld], rot_z [9][ld]   root_rot_mat = quat.toRotationMatrix() and root_rot_mat_z = AngleAxisd(yaw, UnitZ), row-major
 *     x0 [12][ld]                  only rows 0-2 (root_euler = Utils::quat_to_euler, utils/Utils.cpp:7-32) and rows 6-8
 *                                  (root_ang_vel = root_rot_mat * imu_ang_vel, world) are written; rows 3-5 and 9-11 belong to the
 *                                  estimator.  With ld the x0 and rot of an a1mpc_inputs pass as they are.
 *                                  ld applies to rot, rot_z and x0 alike: a1mpc_stance_qp_batch takes rot_z with its ld, but
 *                                  a1mpc_update_plan_batch and a1mpc_swing_legs_batch take a dense rot_z [9][B], so with ld > B
 *                                  write rot_z with a second call (ld = B) or into a separate dense array for them.
 *     imu_acc [3][B], imu_ang_vel [3][B]   the (filtered) readings, as a1mpc_ekf_update_batch takes them; imu_acc needs acc.
 *   As the reference computes it, not as it means it: the quaternion is NOT normalised (Eigen's toRotationMatrix and quat_to_euler
 *   use the raw coefficients); the pitch argument t2 is clamped to +-1 before asin; rot_z is Eigen's AngleAxis matrix of the yaw that
 *   quat_to_euler returned (cos / sin of the full angle, diagonal element (1 - c) + c).  One difference in timing: Gazebo computes
 *   root_ang_vel in the IMU callback with whatever rotation the last pose message left, Isaac in the pose callback with the last gyro
 *   sample; here it always uses the rotation and the gyro sample of the same call.
 *
 * a1mpc_command_batch: main_update's front half (GazeboA1ROS.cpp:117-188, HardwareA1ROS.cpp:98-158, IsaacA1ROS.cpp:75-137).
 *   cmd_state  a1mpc_command_bytes(B) bytes: joy_cmd_body_height, joy_cmd_ctrl_state, root_euler_d,
 *              root_pos_d, kp_linear, root_lin_vel_d and the init parameters.  a1mpc_command_init_batch sets it from cp (batch-uniform):
 *              body_height = the adapter's initial joy_cmd_body_height (0.3 Gazebo, 0.12 hardware, 0.32 Isaac: GazeboA1ROS.h:130,
 *              HardwareA1ROS.h:107, IsaacA1ROS.h:80), the clamp JOY_CMD_BODY_HEIGHT_MIN / _MAX (0.1 / 0.32, A1Params.h:16-17),
 *              kp_linear and kp_linear_lock (120, 120, 500 / 120, 120 from the ROS-parameter defaults, A1CtrlStates.h:270-301) and
 *              the adapter variant; control state 0, everything else zero (A1CtrlStates::reset).  Its ref (may be NULL, ref_ld >= B)
 *              gets those reset values in all nine rows, which is what the first command call reads back (below).
 *   cmd [7][B]  per robot, in physical units (what joy_callback leaves after its axis scaling): velx, vely, velz, roll rate, pitch
 *               rate, yaw rate, toggle request (non-zero = toggle walking).
 *   root_pos [3][root_pos_ld]  the previous estimate (A1BasicEKF.cpp:162): x0 + 3 ld of an a1mpc_inputs passes as it is.
 *   Per tick: height += velz dt, clamped; the walking toggle; root_lin_vel_d.xy = (velx, vely); root_ang_vel_d = the three rates;
 *   root_euler_d[0..1] += rate dt; root_euler_d[2] += yaw rate dt; root_pos_d[2] = height; movement_mode = walking; the step out of
 *   walking locks root_pos_d.xy = root_pos.xy with the lock gains; while walking |root_lin_vel_d.xy| > 0.05 refreshes
 *   root_pos_d.xy = root_pos.xy and zeroes kp_linear.xy, otherwise kp_linear.xy = the lock gains.  The variants differ where the
 *   adapters differ, reproduced literally: only Gazebo sets root_lin_vel_d[2] = velz (GazeboA1ROS.cpp:152); the hardware and Isaac
 *   adapters set x and y only and leave it at 0 (HardwareA1ROS.cpp:121-123, IsaacA1ROS.cpp:99-101).  A1MPC_VARIANT_HARDWARE
 *   also ASSIGNS root_euler_d[0..1] the roll and pitch rates instead of integrating them (HardwareA1ROS.cpp:129-130).
 *   outputs: movement_mode [B] (the layout of a1mpc_update_plan_batch / a1mpc_ekf_update_batch); kp_linear [3][stance_ld] and des
 *   [12][stance_ld] (may be NULL) in the layout of a1mpc_stance_qp_batch (its ld); ref [9][ref_ld] (may be NULL) in the a1mpc_inputs
 *   layout, so root_lin_vel_d is ref + 5 ref_ld for a1mpc_update_plan_batch.
 *   The pitch round trip: compute_grf's terrain adaptation overwrites root_euler_d[1] (a1mpc_terrain_pitch_batch writes row 1 of ref,
 *   A1RobotControl.cpp:358-364) and the next main_update integrates on top of it.  So when ref is given, this tick's root_euler_d[1]
 *   starts from what row 1 of ref holds; without ref it starts from the state.  Pass the same ref to a1mpc_command_init_batch (or
 *   hold 0 in its row 1) before the first call.
 * A1MPC_EINVAL: NULL handle, state or mandatory array, B <= 0, an ld < B, a state buffer that is not device memory, unknown variant. */
#define A1MPC_VARIANT_GAZEBO   0
#define A1MPC_VARIANT_HARDWARE 1
#define A1MPC_VARIANT_ISAAC    2
typedef struct a1mpc_command_params {
  int    variant;               /* A1MPC_VARIANT_* */
  double body_height;           /* initial joy_cmd_body_height */
  double body_height_min, body_height_max;
  double kp_linear[3];          /* initial kp_linear */
  double kp_linear_lock[2];     /* kp_linear_lock_x, _y */
} a1mpc_command_params;
size_t a1mpc_imu_bytes(int B);
int  a1mpc_imu_init_batch(a1mpc_handle* h, int B, void* imu_state);
int  a1mpc_orientation_batch(a1mpc_handle* h, int B, const double* quat, const double* gyro, const double* acc, void* imu_state, double* rot,
                             double* rot_z, double* x0, size_t ld, double* imu_acc, double* imu_ang_vel);
size_t a1mpc_command_bytes(int B);
int  a1mpc_command_init_batch(a1mpc_handle* h, int B, void* cmd_state, const a1mpc_command_params* cp, double* ref, size_t ref_ld);
int  a1mpc_command_batch(a1mpc_handle* h, int B, void* cmd_state, double dt, const double* cmd, const double* root_pos, size_t root_pos_ld,
                         uint32_t* movement_mode, double* kp_linear, double* ref, size_t ref_ld, double* des, size_t stance_ld);

/* ---- a whole control tick in one call: raw sensor arrays in, joint torques out ---------------------------------------------
 * A tick object owns the controller state of B robots (IMU filters, command state, gait counters, swing state, EKF, warm-start faces,
 * the previous torques) and every intermediate array, and runs the stages above in the order of one main_update + compute_grf +
 * compute_joint_torques pass:
 *   1 orientation (the IMU filters of the Gazebo and Isaac adapters; none for A1MPC_VARIANT_HARDWARE)   2 leg kinematics   3 command
 *   4 update_plan   5 swing legs   6 EKF: a1mpc_ekf_init_batch on the first run after create or reset, the update after that; a robot
 *     reset by a1mpc_tick_reset_robots since the last run gets the init instead of the update (its x0 rows 3-5 and 9-11 stay zero on
 *     that run, as on a fresh tick's first run)
 *   7 A1MPC_TICK_MPC: terrain pitch, then the MPC solve, posed one of two ways by gait.horizon:
 *     0 (the default): the contact pattern held over the horizon as compute_grf poses it: the solve of a1mpc_solve_batch_warm with
 *       shift 0 (horizon 10) or the cold a1mpc_solve_batch (horizon 20).  It takes part in the fused collect (a1mpc_peer_gather_*) exactly
 *       as a1mpc_solve_batch_warm does.
 *     the handle's horizon N: the scheduled tick, an extension beyond the reference.  The solve sees the gait's planned contacts over the
 *       horizon: the solve of a1mpc_solve_batch_ext_warm with shift 1 (horizon 10) or the cold a1mpc_solve_batch_ext (horizon 20) on the
 *       schedule [N][B] of a1mpc_update_plan_batch, whose step 0 is replaced by the swing stage's contacts (plan OR early contact: the
 *       feet the torque stage treats as stance), world-z friction pyramids (no normals).  Like a1mpc_solve_batch_ext it does not take
 *       part in the fused collect.  The schedule stays inside the tick.
 *     Either way the friction pyramids stand on world z unless a1mpc_tick_set_terrain chose another source (below).
 *     A1MPC_TICK_QP: a1mpc_stance_qp_batch (world-z pyramids unless a1mpc_tick_set_stance_terrain chose another source, below).
 *   8 joint torques.
 * The arrays connect as in a hand-built chain of those entry points: x0 rows 3-5 / 9-11 are the EKF's estimate (zero until its first
 * update), update_plan's root_lin_vel_d is ref row 5 (MPC) or des row 6 (QP), and in MPC mode the command stage reads ref row 1 back, so
 * the terrain pitch of one tick is what the next tick integrates on.  Stages 1-3 and 4-5 run fused, two kernels with one thread per
 * robot; their results are bit-identical to the staged kernels.
 *
 * Batch-major, ld = B, either all-host or all-device arrays in one call (host: the call copies and synchronises; device: it only enqueues,
 * allocates nothing and does not synchronise):
 *   in:  quat [4][B] (w, x, y, z), gyro [3][B], acc [3][B], joint_pos [12][B], joint_vel [12][B], foot_force [4][B] (already filtered),
 *        cmd [7][B] (as a1mpc_command_batch), gait_counter_speed [4][B]
 *   out: tau [12][B] (mandatory; an entry whose new value is NaN keeps the previous one), f_body [12][B] (foot_forces_grf), status [B] (the
 *        solve's or the stance QP's), contacts [B], movement_mode [B], x0 [12][B], ref [9][B] (MPC mode only; NULL in QP mode).  Any but tau
 *        may be NULL.
 * create and reset put the state where a chain starts: zero x0, gait counters and tau; a1mpc_imu_init_batch, a1mpc_command_init_batch (with
 * ref in MPC mode), a1mpc_swing_init_batch and a1mpc_warm_reset.  create also sizes the handle's scratch for B (the scheduled tick's
 * too).  Destroy a tick before its handle.  A1MPC_EINVAL: precision 32 (these stages are fp64), an unknown mode or variant, in MPC mode a
 * gait.horizon other than 0 or the handle's horizon, B <= 0, dt <= 0, counter_per_swing <= 0, a mix of host and device arrays, ref in QP
 * mode. */
#define A1MPC_TICK_QP  0   /* stance_leg_control_type 0 */
#define A1MPC_TICK_MPC 1   /* stance_leg_control_type 1 */
typedef struct a1mpc_tick a1mpc_tick;
typedef struct a1mpc_tick_params {
  int mode;                       /* A1MPC_TICK_QP | A1MPC_TICK_MPC */
  int use_terrain_adapt;          /* MPC mode: terrain pitch written into root_euler_d[1] */
  int assume_flat_ground;         /* the EKF's foot-height measurement */
  a1mpc_gait_params gait;         /* MPC mode: horizon 0 = the held pattern, N = the handle's horizon = the scheduled tick; QP mode: unused */
  a1mpc_command_params command;   /* its variant also selects the IMU filters: none for A1MPC_VARIANT_HARDWARE */
  double rho_opt[12], rho_fix[20];               /* a1mpc_leg_kinematics_batch */
  double kp_foot[12], kd_foot[12];               /* a1mpc_swing_legs_batch */
  double km_foot[3], torques_gravity[12];        /* a1mpc_joint_torques_batch */
  double kd_linear[3], kp_angular[3], kd_angular[3];   /* QP mode: a1mpc_stance_qp_batch */
} a1mpc_tick_params;
typedef struct a1mpc_tick_inputs {
  const double *quat, *gyro, *acc, *joint_pos, *joint_vel, *foot_force, *cmd, *gait_counter_speed;
} a1mpc_tick_inputs;
typedef struct a1mpc_tick_outputs {
  double* tau;
  double* f_body;
  int32_t* status;
  uint32_t* contacts;
  uint32_t* movement_mode;
  double* x0;
  double* ref;
} a1mpc_tick_outputs;
/* the reference's launch parameters of one adapter (config/{gazebo,hardware,isaac}_a1_{qp,mpc}.yaml, A1CtrlStates.h, A1Params.h, the adapters'
 * leg geometry); A1MPC_EINVAL for an unknown variant or mode */
int  a1mpc_default_tick_params(int variant, int mode, a1mpc_tick_params* tp);
int  a1mpc_tick_create(a1mpc_handle* h, int B, const a1mpc_tick_params* tp, a1mpc_tick** out);
int  a1mpc_tick_reset(a1mpc_tick* t);
/* Put the robots b with mask[b] != 0 back where a1mpc_tick_create / a1mpc_tick_reset put them; every other robot's state is untouched, so
 * a simulator can restart one environment's episode while the rest of the batch keeps walking.  mask [B] (uint8: a numpy / torch bool
 * array passes as is), host or device memory.  Device: enqueued only, no allocation, no synchronisation.  Host: copied, then the same,
 * and the call synchronises.  The next a1mpc_tick_run initialises the EKF of the reset robots instead of updating it, exactly as the
 * first run after create does for all robots.  Several calls before one run reset the union of their masks; a1mpc_tick_reset
 * supersedes a pending partial reset; an all-zero mask changes nothing.  A1MPC_EINVAL: a NULL tick or mask. */
int  a1mpc_tick_reset_robots(a1mpc_tick* t, const uint8_t* mask);
/* Where an MPC-mode tick's friction pyramids stand (stage 7).  The ground can only push inside a cone about its own normal, so on a slope
 * the world-z pyramid is the wrong constraint.
 *   A1MPC_TERRAIN_FLAT       world z, the default: the tick as if this call had never been made (normals ignored).
 *   A1MPC_TERRAIN_ESTIMATED  the normal of the walking surface the terrain stage fits every tick (a1mpc_terrain_normals_batch), the same
 *                            for all four feet.
 *   A1MPC_TERRAIN_GIVEN      normals [12][B]: a caller-owned DEVICE array (per foot, world frame, n_z > 0, e.g. a height-field lookup)
 *                            that every later run reads at stage 7; the caller orders its writes before the run, as with any device
 *                            input.  The terrain stage still runs and writes ref row 1 as before.
 * With ESTIMATED or GIVEN, stage 7 is a1mpc_terrain_normals_batch and then the solve of a1mpc_solve_batch_ext_warm with those normals:
 * on the scheduled tick's schedule with shift 1; with the held pattern on a schedule of the swing stage's contacts in all N rows with
 * shift 0 (the cold a1mpc_solve_batch_ext at horizon 20).  Like every _ext solve it does not take part in the fused collect.  Switching
 * source between runs needs no clean-up: the warm slots of the held-pattern solve and of the _ext solve read each other as "no guess".
 * The first call to a non-flat source allocates the tick's normals and held schedule and sizes the handle's scratch (it may
 * synchronise); after it a run on device arrays still allocates nothing and does not synchronise.  a1mpc_tick_reset and
 * a1mpc_tick_reset_robots keep the source.  A1MPC_EINVAL: a NULL tick, an unknown source, a non-flat source in QP mode (a QP-mode tick
 * takes a1mpc_tick_set_stance_terrain below) or on a handle with non-isotropic r, GIVEN with a NULL or host pointer. */
#define A1MPC_TERRAIN_FLAT      0
#define A1MPC_TERRAIN_ESTIMATED 1
#define A1MPC_TERRAIN_GIVEN     2
int  a1mpc_tick_set_terrain(a1mpc_tick* t, int source, const double* normals);
/* Where a QP-mode tick's stance friction pyramids stand (stage 7), with the sources of a1mpc_tick_set_terrain:
 *   A1MPC_TERRAIN_FLAT       world z, the default: the tick as if this call had never been made (normals ignored).
 *   A1MPC_TERRAIN_ESTIMATED  the walking surface's normal (a1mpc_surface_normals_batch) from the recent-contact points the swing stage
 *                            records, the same for all four feet.
 *   A1MPC_TERRAIN_GIVEN      normals [12][B]: a caller-owned DEVICE array (per foot, world frame, n_z > 0) that every later run reads at
 *                            stage 7; the caller orders its writes before the run.
 * With ESTIMATED or GIVEN, stage 7 is a1mpc_surface_normals_batch (ESTIMATED only) and then a1mpc_stance_qp_batch_ext with those normals.
 * Stage 7 writes nothing else: the reference adapts to terrain only in MPC mode, so no terrain filter advances and des is untouched.  The
 * first call to a non-flat source allocates the tick's normals (it may synchronise); after it a run on device arrays allocates nothing and
 * does not synchronise.  a1mpc_tick_reset and a1mpc_tick_reset_robots keep the source.  A1MPC_EINVAL: a NULL tick, an MPC-mode tick (it
 * takes a1mpc_tick_set_terrain), an unknown source, GIVEN with a NULL or host pointer. */
int  a1mpc_tick_set_stance_terrain(a1mpc_tick* t, int source, const double* normals);
/* Run an MPC-mode tick's solve at a lower rate than the tick.  The reference computes its ground forces in a thread of its own and the
 * torque loop applies whatever forces that thread wrote last; here each robot solves on every period-th run, staggered across the batch,
 * so that a run solves about B / period QPs instead of B.
 *   Which robots solve: n_b counts robot b's runs since its start (create, a1mpc_tick_reset, its own a1mpc_tick_reset_robots or the
 *   last a1mpc_tick_set_mpc_period).  Robot b solves on run n_b when n_b == 0 || n_b % period == b % period.  j_b, the runs since robot
 *   b's last solve, stays in [0, period - 1].
 *   On a robot's solve run, f_body and status come from the solve as on a plain tick.  On its other runs:
 *     A1MPC_PLAYBACK_HOLD  f_body and status stay as its last solve wrote them (the reference's torque thread); nothing runs for it.
 *     A1MPC_PLAYBACK_PLAN  f_body = R^T u_j with this run's R (rot) and u_j the world-frame forces of step j_b of its last solve's plan
 *                          (u_full); status stays.  The plan advances one horizon step per run, which assumes that the handle's dt is the
 *                          tick's period, as in the reference (mpc_dt = control period = 2.5 ms, a1mpc_default_config).
 *   The torque stage uses this run's contacts either way: a force planned for a foot that has since lifted is not applied.
 * The warm start keeps its shift on the held pattern (0, a guess `period` runs old is only a worse guess); the scheduled tick takes
 * shift = period, as a due robot's stored faces are `period` schedule steps old.  A multi-rate tick does not take part in the fused
 * collect.  period = 1 is the tick as if this call had never been made.  Every call makes every robot solve on its next run; the resets
 * keep the period and the playback.  The first call with period > 1 allocates the tick's counters (and, for PLAN, its plan [12 N][B])
 * and may synchronise; after it a run on device arrays still allocates nothing and does not synchronise.  A1MPC_EINVAL: a NULL tick,
 * QP mode (the stance QP runs on every run), period outside [1, N] (N the handle's horizon), an unknown playback. */
#define A1MPC_PLAYBACK_HOLD 0   /* between solves: f_body and status of the robot's last solve, unchanged */
#define A1MPC_PLAYBACK_PLAN 1   /* between solves: R_now^T * u_j, step j of the last solve's world-frame plan */
int  a1mpc_tick_set_mpc_period(a1mpc_tick* t, int period, int playback);
/* The playback of A1MPC_PLAYBACK_PLAN as a staged entry point: rot [9][B], u_full [12 N][B] (as a1mpc_outputs.u_full), step [B] in,
 * f_body [12][B] in/out, host or device.  step_b = 0 leaves robot b's f_body untouched (that run's solve wrote it); 1 <= step_b < N writes
 * f_body = R^T u_full[12 step_b : 12 step_b + 12]; step_b >= N writes zero forces.  A1MPC_EINVAL: NULL handle or array, B <= 0. */
int  a1mpc_plan_forces_batch(a1mpc_handle* h, int B, const double* rot, const double* u_full, const uint32_t* step, double* f_body);
/* Give each robot of a tick its own gait (both modes): gait [6][B], the rows of a1mpc_gait_row / a1mpc_update_plan_gait_batch, host or
 * device.  The rows are checked on the device and copied into the tick; the call synchronises (twice: after the check, and after the
 * copy, so that it returns with the rows in the tick and the caller may rewrite or free its array at once, from any stream).  A bad row gives A1MPC_EINVAL naming
 * the first bad robot and the rule it breaks, and the previous gaits stay in force.  gait = NULL returns to the reference's trot (tp.gait's
 * cpg and cps, offsets 0 120 120 0): a tick that never made this call, or made it with NULL, runs exactly as before.
 *   cps and cpg apply from the next run.  The offsets apply when a robot stands, where the reference calls gait_counter_reset(): a walking
 *   robot keeps its leg phases until it stops (no gait-transition planner).
 *   a1mpc_tick_reset and a1mpc_tick_reset_robots keep the gaits.  A reset robot starts in standstill (joy_cmd_ctrl_state 0), so unless its
 *   first run's cmd toggles walking it takes its row's offsets on that run.  To re-phase robots: set the gaits, then reset those robots; or,
 *   without a reset, toggle them to standstill for one run with cmd row 6 and back to walking on a later run.
 *   The first non-NULL call allocates 6 B doubles in the tick; after it a run on device arrays allocates nothing and does not synchronise.
 *   A pronk's flight phase gives robots with no stance foot: they take the existing no-contact path (A1MPC_STATUS_NO_CONTACT, zero
 *   forces) in both modes.
 * A1MPC_EINVAL: a NULL tick, a bad row. */
int  a1mpc_tick_set_gaits(a1mpc_tick* t, const double* gait);
int  a1mpc_tick_run(a1mpc_tick* t, double dt, const a1mpc_tick_inputs* in, const a1mpc_tick_outputs* out);
int  a1mpc_tick_destroy(a1mpc_tick* t);

/* ---- device memory, stream and timing helpers (so hosts need no CUDA headers) -------------- */
int  a1mpc_device_alloc(a1mpc_handle* h, size_t bytes, void** ptr);
int  a1mpc_device_free(a1mpc_handle* h, void* ptr);
int  a1mpc_host_alloc(a1mpc_handle* h, size_t bytes, void** ptr);   /* pinned */
int  a1mpc_host_free(a1mpc_handle* h, void* ptr);
int  a1mpc_memcpy_h2d(a1mpc_handle* h, void* dst, const void* src, size_t bytes);  /* async on the stream */
int  a1mpc_memcpy_d2h(a1mpc_handle* h, void* dst, const void* src, size_t bytes);  /* async on the stream */
int  a1mpc_sync(a1mpc_handle* h);
int  a1mpc_event_create(a1mpc_handle* h, void** ev);
int  a1mpc_event_destroy(a1mpc_handle* h, void* ev);
int  a1mpc_event_record(a1mpc_handle* h, void* ev);                  /* on the handle's stream */
int  a1mpc_event_elapsed_ms(a1mpc_handle* h, void* start, void* stop, float* ms); /* syncs on stop */
/* number of kernels this handle has launched since creation (bench.py's gpu_launches) */
int64_t a1mpc_launch_count(const a1mpc_handle* h);
/* measured peak of the fp64 FMA pipe on this device, TFLOP/s (dependent-free DFMA stream) */
int  a1mpc_measure_fp64_peak(a1mpc_handle* h, double* tflops);
/* Per-class kernel timing for roofline reports: between begin and end every a1mpc_solve_batch records a
 * CUDA-event pair around each class kernel ON THE STREAM THAT KERNEL RUNS ON (up to max_calls calls).
 * end() synchronises and returns the summed device time in ms of the kernels for 1,2,3,4 stance feet. */
int  a1mpc_profile_begin(a1mpc_handle* h, int max_calls);
int  a1mpc_profile_end(a1mpc_handle* h, double* ms_per_class4, int* calls);
/* writes one buffer larger than L2 (flushes L2 between timed iterations when asked to) */
int  a1mpc_flush_l2(a1mpc_handle* h);

/* ---- optional final collect across GPUs (SURVEY 8e): all-gather of f_body over NCCL ------- */
/* NCCL is dlopen'ed at first use; without it these return A1MPC_ENCCL and nothing else in the
 * library depends on it.  unique_id is a 128-byte ncclUniqueId produced on rank 0. */
int  a1mpc_nccl_unique_id(void* unique_id128);
int  a1mpc_nccl_init(a1mpc_handle* h, int nranks, int rank, const void* unique_id128);
/* gathers f_local [12][B_local] (device) from every rank into f_all [nranks][12][B_local].  Asynchronous: the collective runs on
 * the handle's collect stream after everything enqueued so far and overlaps later solves; a1mpc_sync and a1mpc_event_record
 * wait for it.  Do not overwrite f_local / read f_all before one of them. */
int  a1mpc_allgather_forces(a1mpc_handle* h, const double* f_local, double* f_all, int B_local);

/* ---- fused final collect (SURVEY 2.3 last row / 8e): the solve kernels store the forces into every GPU's gathered buffer -------
 * One process per GPU.  Each rank allocates its gathered buffer f_all [nranks][B_local][12] (QP-major: the 12 body-frame forces of a
 * robot are contiguous, leg-major -- NOT the batch-major layout of f_body / ncclAllGather) with a1mpc_peer_gather_create, which
 * returns a 64-byte CUDA IPC handle; the ranks exchange the handles (any transport: the caller's MPI / torch.distributed / files)
 * and map each other's buffers with a1mpc_peer_gather_connect.  From then on every a1mpc_solve_batch / _warm call with device
 * pointers and B == B_local ALSO stores the 12 forces of every QP, straight from the solve kernels' epilogue, into block [rank] of
 * every rank's buffer (one contiguous 96-byte peer store per QP and rank over NVLink / NVSwitch -- no collective call, no extra pass
 * over the data) and then
 * publishes the call's sequence number to every rank.  a1mpc_peer_gather_wait enqueues, on the handle's collect stream (forked after
 * everything enqueued so far, so that later solves are not held back by a slower peer; a1mpc_sync and a1mpc_event_record join
 * it, exactly like the NCCL collect), a wait until the forces of this rank's latest call number have arrived from ALL ranks
 * (the ranks must make the same sequence of calls).
 * Semantics: "latest value" -- a rank that runs ahead overwrites its block with its next call's forces; callers that must consume
 * call k everywhere before any rank starts call k+1 add their own barrier.  precision 32: the buffer holds float.
 * The wait itself is a stream memory operation (cuStreamWaitValue64 on this rank's flag array: no SM is occupied); where the driver
 * refuses it, or with A1MPC_PEER_WAIT_KERNEL=1, a one-warp polling kernel with a ~2 s cap is used instead, and a peer that never
 * arrives is then reported by a1mpc_peer_gather_status (0 = fine, r+1 = rank r timed out) instead of hanging the stream.
 * Needs peer access between the GPUs (same NVLink domain) and CUDA IPC between the processes; A1MPC_ECUDA otherwise -- the NCCL
 * all-gather above remains available as the portable path. */
int  a1mpc_peer_gather_create(a1mpc_handle* h, int nranks, int rank, int B_local, void* ipc_handle64);
int  a1mpc_peer_gather_connect(a1mpc_handle* h, const void* all_handles /* nranks x 64 bytes, rank order */);
int  a1mpc_peer_gather_buffer(a1mpc_handle* h, double** f_all);
int  a1mpc_peer_gather_wait(a1mpc_handle* h);
int  a1mpc_peer_gather_status(a1mpc_handle* h, int* timed_out_rank_plus_1);
int  a1mpc_peer_gather_destroy(a1mpc_handle* h);

/* ---- synthetic workload generator (SURVEY 8d), host-side, deterministic ------------------- */
/* Fills host SoA arrays (ld = B) with the trot-gait state distribution of the benchmark.
 * config_id: 2 = trot narrow noise (configs 2,3,5), 4 = wide noise (config 4's state noise).
 * seed = 0xA1C0FFEE + config_id + `stream` (use the rank / batch index as stream). */
int  a1mpc_gen_states(int config_id, uint64_t stream, int B, double* x0, double* rot, double* foot,
                      double* ref, uint32_t* contact);
/* config-4 extras for the same (config_id, stream, B): per-step schedules [N][B] drawn from trot / bound / rotary gallop at
 * a random phase of a 16-step period, and per-foot normals [12][B] = z tilted by N(0,0.2) rad about a random horizontal axis */
int  a1mpc_gen_schedule(int config_id, uint64_t stream, int B, int horizon, uint32_t* contact_sched, double* normals);

#ifdef __cplusplus
}
#endif
#endif /* A1MPC_H_ */
