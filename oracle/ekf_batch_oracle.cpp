// oracle/ekf_batch_oracle.cpp -- TEST INFRASTRUCTURE, not product code.
//
// oracle_ekf_update (a1mpc_oracle.cpp, the dense long-double restatement of A1BasicEKF::update_estimation, pinned to the reference's
// own A1BasicEKF by tests/test_ref_pin.py) for a batch of robots on host threads, in the layout of a1mpc_ekf_update_batch.  The
// per-robot body is called as it is, from liba1mpc_oracle.so; one robot-tick costs about 0.2 ms on one core, so the long filter
// runs of tests/test_gpu_ekf.py need the threads.  Built by `make -C oracle -f ekf_batch.mk` (the top-level Makefile runs it).
#include <atomic>
#include <cstddef>
#include <cstdint>
#include <thread>
#include <vector>

extern "C" {

int oracle_ekf_update(double dt, int assume_flat_ground, uint32_t movement_mode, const double* imu_acc, const double* imu_ang_vel,
                      const double* rot, const double* foot_pos_rel, const double* foot_vel_rel, const double* foot_force, double* x, double* P,
                      double* root_pos, double* root_lin_vel, uint32_t* est_contacts);

// state [B][342] (x[18], P[18][18] row-major per robot) in/out, movement_mode [B], imu_acc [3][B], imu_ang_vel [3][B], rot [9][B],
// foot_pos_rel [12][B], foot_vel_rel [12][B], foot_force [4][B] (ld = B); out (any may be NULL) root_pos [3][B], root_lin_vel [3][B],
// est_contacts [B], rc [B].  A robot whose rc is not 0 keeps its state and has none of its outputs written.
int oracle_ekf_update_batch(int B, double dt, int assume_flat_ground, const uint32_t* movement_mode, const double* imu_acc,
                            const double* imu_ang_vel, const double* rot, const double* foot_pos_rel, const double* foot_vel_rel,
                            const double* foot_force, int nthreads, double* state, double* root_pos, double* root_lin_vel,
                            uint32_t* est_contacts, int32_t* rc) {
  if (nthreads < 1) nthreads = 1;
  std::atomic<int> next(0);
  auto work = [&]() {
    for (;;) {
      const int b = next.fetch_add(1);
      if (b >= B) break;
      const size_t ld = (size_t)B;
      double acc[3], gyro[3], R[9], fk[12], fv[12], ff[4], pos[3], vel[3];
      for (int k = 0; k < 3; ++k) { acc[k] = imu_acc[k * ld + b]; gyro[k] = imu_ang_vel[k * ld + b]; }
      for (int k = 0; k < 9; ++k) R[k] = rot[k * ld + b];
      for (int k = 0; k < 12; ++k) { fk[k] = foot_pos_rel[k * ld + b]; fv[k] = foot_vel_rel[k * ld + b]; }
      for (int k = 0; k < 4; ++k) ff[k] = foot_force[k * ld + b];
      double* x = state + (size_t)b * (18 + 18 * 18);
      uint32_t ec = 0;
      const int r = oracle_ekf_update(dt, assume_flat_ground, movement_mode[b], acc, gyro, R, fk, fv, ff, x, x + 18, pos, vel, &ec);
      if (rc) rc[b] = r;
      if (r) continue;
      for (int k = 0; k < 3; ++k) {
        if (root_pos) root_pos[k * ld + b] = pos[k];
        if (root_lin_vel) root_lin_vel[k * ld + b] = vel[k];
      }
      if (est_contacts) est_contacts[b] = ec;
    }
  };
  if (nthreads == 1) { work(); return 0; }
  std::vector<std::thread> th;
  for (int t = 0; t < nthreads; ++t) th.emplace_back(work);
  for (auto& t : th) t.join();
  return 0;
}

}  // extern "C"
