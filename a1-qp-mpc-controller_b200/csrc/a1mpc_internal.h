// a1mpc_internal.h -- host-side glue between the translation units of liba1mpc.so
#pragma once
#include <cuda_runtime.h>
#include "a1mpc_device.cuh"

namespace a1mpc {

struct ClassLaunch {
  int wpc = 1;
  size_t smem = 0;
  int max_ctas = 0;  // resident CTAs on the whole device (persistent grid size)
  bool supported = false;
};

// fused path (a1mpc_solve_n10.cu / a1mpc_solve_n20.cu)
cudaError_t fused_setup_n10(int sm_count, ClassLaunch (&cls)[5]);
cudaError_t fused_setup_n20(int sm_count, ClassLaunch (&cls)[5]);
void fused_launch_n10(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out);
void fused_launch_n20(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out);
// warm-started variant of the N = 10 classes (a1mpc_solve_batch_warm); set up by fused_setup_n10
void fused_launch_n10_warm(int ns, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count,
                           const DevOutputs& out, uint32_t* warm, int shift);
// extended path (per-step contact schedules + terrain normals), a1mpc_solve_ext.cu
cudaError_t ext_setup(int horizon, int sm_count, ClassLaunch& c);
void ext_launch(int horizon, const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out);
// compacted two-stance-feet-per-step class of the extended path (a1mpc_sched.cuh; opt-in, N = 10)
cudaError_t sched2_setup(int sm_count, ClassLaunch& c);
void sched2_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out);
// warm-started variants of both (a1mpc_solve_batch_ext_warm, N = 10)
cudaError_t ext_warm_setup(int sm_count, ClassLaunch& c);
void ext_warm_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out,
                     uint32_t* warm, int shift);
cudaError_t sched2_warm_setup(int sm_count, ClassLaunch& c);
void sched2_warm_launch(const ClassLaunch& c, cudaStream_t st, int B, const DevParams& P, const double* rec, const int* count, const DevOutputs& out,
                        uint32_t* warm, int shift);
cudaError_t build_dense_launch(const DevParams& P, const DevInputs& in, int B, double* H, double* g, double* lb, double* ub, cudaStream_t st);

// QP-major side entry points (a1mpc_dense.cu)
cudaError_t dense_setup(int horizon);
// scratch: (4*B + 8) ints
cudaError_t dense_qp_mats_launch(const DevParams& P, int B, const double* A_d, const double* B_d_list, const double* x0, const double* x_d,
                                 double* H, double* g, double* A_qp, double* B_qp, cudaStream_t st);
// returns cudaErrorInvalidValue for configurations whose factor does not fit (N=20 with >2 stance feet)
cudaError_t dense_solve_launch(const DevParams& P, int sm_count, int B, const double* H, const double* g, const uint32_t* contact, double* u,
                               int32_t* status, int* scratch, cudaStream_t st, int* nlaunch);
cudaError_t grf_qp_launch(int sm_count, int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot,
                          const uint32_t* contact, double* f_body, int32_t* status, int* scratch, cudaStream_t st, int* nlaunch);
// the same QP with the PD law in front of it, batch-major arrays with leading dimension ld (a1mpc_stance_qp_batch);
// gains9 = kd_linear, kp_angular, kd_angular (host); scratch: stance_scratch_bytes(B) bytes of device memory.  normals [12][ld] (device)
// poses each stance foot's pyramid on its terrain normal (a1mpc_stance_qp_batch_ext); NULL: world z
size_t stance_scratch_bytes(int B);
cudaError_t stance_qp_launch(int sm_count, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                             const uint32_t* contact, const double* des, const double* kp_linear, const double* gains9, double mass,
                             const double* normals, double* f_body, int32_t* status, double* root_acc, void* scratch, cudaStream_t st,
                             int* nlaunch);

// orientation and command stages (a1mpc_command.cu, kernels in a1mpc_command.cuh), thread per robot on the stream
size_t imu_state_doubles();       // per robot
size_t command_state_doubles();   // per robot
cudaError_t imu_init_launch(int B, double* state, cudaStream_t st);
cudaError_t orientation_launch(int B, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                               double* euler, double* ang_vel, size_t ld, double* imu_acc, double* imu_ang_vel, cudaStream_t st);
cudaError_t command_init_launch(int B, const a1mpc_command_params& cp, double* state, double* ref, size_t ref_ld, cudaStream_t st);
cudaError_t command_launch(int B, double dt, double* state, const double* cmd, const double* root_pos, size_t pos_ld, uint32_t* movement_mode,
                           double* kp, double* ref, size_t ref_ld, double* des, size_t des_ld, cudaStream_t st);
// the fused front of a control tick (a1mpc_tick_run): both stages above in one thread per robot, every array dense (ld = B); x0 [12][B]
// (rows 0-2 and 6-8 written, rows 3-5 read as root_pos); imu null = unfiltered; ref null in QP mode
cudaError_t tick_front_a_launch(int B, double dt, const double* quat, const double* gyro, const double* acc, double* imu, double* rot, double* rot_z,
                                double* x0, double* imu_acc, double* imu_ang_vel, double* cmd_state, const double* cmd, uint32_t* movement_mode,
                                double* kp, double* ref, double* des, cudaStream_t st);

}  // namespace a1mpc
