// oracle/command_oracle.cpp -- TEST INFRASTRUCTURE, not product code: the oracle of a1mpc_orientation_batch / a1mpc_command_batch.
// Built by `make -C oracle -f command.mk` into oracle/liba1mpc_command_oracle.so, bound by oracle/command_oracle_py.py.  Nothing under
// a1-qp-mpc-controller_b200/ may include, link or call this file.  Dependency-free C++17.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <vector>

// ---------------------------------------------------------------------------------------------------------------------
// Orientation stage: the IMU / pose callbacks of the adapters (GazeboA1ROS.cpp:235-299, HardwareA1ROS.cpp:262-276,
// IsaacA1ROS.cpp:183-241) restated per robot: Eigen's Quaternion::toRotationMatrix, Utils::quat_to_euler (utils/Utils.cpp:7-32),
// Eigen's AngleAxis::toRotationMatrix about UnitZ, root_ang_vel = root_rot_mat * imu_ang_vel, and the MovingWindowFilter(5) of
// acc and gyro (utils/filter.hpp) as std::deque windows.  quat_to_euler and the filter are PINNED to the reference's own compiled code
// by tests/test_command_ref_pin.py.
//
// Command stage: main_update's front half (GazeboA1ROS.cpp:117-188, HardwareA1ROS.cpp:98-158, IsaacA1ROS.cpp:75-137), restated:
// those bodies need ROS message types and cannot be compiled here.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct Window {   // MovingWindowFilter (utils/filter.hpp)
  size_t n;
  std::deque<double> q;
  double sum = 0.0, corr = 0.0;
  explicit Window(size_t n_) : n(n_) {}
  void add(double v) {
    const double t = sum + v;
    if (std::fabs(sum) >= std::fabs(v)) corr += (sum - t) + v;
    else corr += (v - t) + sum;
    sum = t;
  }
  double average(double v) {
    if (q.size() >= n) { add(-q.front()); q.pop_front(); }
    add(v);
    q.push_back(v);
    return (sum + corr) / double(n);
  }
};

void quat_to_euler(double w, double x, double y, double z, double* e) {   // Utils.cpp:7-32, coefficients as given
  const double y_sqr = y * y;
  const double t0 = +2.0 * (w * x + y * z);
  const double t1 = +1.0 - 2.0 * (x * x + y_sqr);
  e[0] = std::atan2(t0, t1);
  double t2 = +2.0 * (w * y - z * x);
  t2 = t2 > +1.0 ? +1.0 : t2;
  t2 = t2 < -1.0 ? -1.0 : t2;
  e[1] = std::asin(t2);
  const double t3 = +2.0 * (w * z + x * y);
  const double t4 = +1.0 - 2.0 * (y_sqr + z * z);
  e[2] = std::atan2(t3, t4);
}

void quat_to_rot(double w, double x, double y, double z, double* r) {   // Eigen QuaternionBase::toRotationMatrix, row-major
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  r[0] = 1 - (tyy + tzz); r[1] = txy - twz; r[2] = txz + twy;
  r[3] = txy + twz; r[4] = 1 - (txx + tzz); r[5] = tyz - twx;
  r[6] = txz - twy; r[7] = tyz + twx; r[8] = 1 - (txx + tyy);
}

void yaw_to_rot_z(double angle, double* r) {   // Eigen AngleAxis::toRotationMatrix with axis (0, 0, 1)
  const double ax[3] = {0.0, 0.0, 1.0};
  const double s = std::sin(angle), c = std::cos(angle);
  const double sa[3] = {s * ax[0], s * ax[1], s * ax[2]};
  const double ca[3] = {(1 - c) * ax[0], (1 - c) * ax[1], (1 - c) * ax[2]};
  double tmp = ca[0] * ax[1];
  r[1] = tmp - sa[2]; r[3] = tmp + sa[2];
  tmp = ca[0] * ax[2];
  r[2] = tmp + sa[1]; r[6] = tmp - sa[1];
  tmp = ca[1] * ax[2];
  r[5] = tmp - sa[0]; r[7] = tmp + sa[0];
  r[0] = ca[0] * ax[0] + c; r[4] = ca[1] * ax[1] + c; r[8] = ca[2] * ax[2] + c;
}

struct Imu {
  bool filtered;
  std::vector<Window> f;   // per robot: acc x, y, z, gyro x, y, z
  Imu(int B, bool filt) : filtered(filt), f(filt ? 6 * (size_t)B : 0, Window(5)) {}
};

struct Command {   // the adapter's joystick state and the A1CtrlStates fields main_update carries
  int variant;
  double hmin, hmax, lock[2];
  std::vector<double> height, euler_d, pos_d, kp, lin_vel_d;
  std::vector<int> ctrl;
};
}  // namespace

extern "C" {

// quat [4][n] (w, x, y, z) -> euler [3][n]
int oracle_quat_to_euler(int n, const double* quat, double* euler) {
  for (int b = 0; b < n; ++b) {
    double e[3];
    quat_to_euler(quat[b], quat[n + b], quat[2 * n + b], quat[3 * n + b], e);
    for (int a = 0; a < 3; ++a) euler[a * n + b] = e[a];
  }
  return 0;
}

// one MovingWindowFilter(W) over T samples x[T] -> averages y[T]
int oracle_window(int W, int T, const double* x, double* y) {
  Window w(W);
  for (int t = 0; t < T; ++t) y[t] = w.average(x[t]);
  return 0;
}

void* oracle_imu_new(int B, int filtered) { return new Imu(B, filtered != 0); }
void oracle_imu_free(void* h) { delete static_cast<Imu*>(h); }

// a1mpc_orientation_batch with every array dense [F][B]; acc may be null (then imu_acc is not written)
int oracle_orientation(void* h, int B, const double* quat, const double* gyro, const double* acc, double* rot, double* rot_z, double* euler,
                       double* ang_vel, double* imu_acc, double* imu_ang_vel) {
  Imu& I = *static_cast<Imu*>(h);
  for (int b = 0; b < B; ++b) {
    double g[3];
    for (int a = 0; a < 3; ++a) {
      const double v = gyro[a * B + b];
      g[a] = I.filtered ? I.f[6 * (size_t)b + 3 + a].average(v) : v;
      imu_ang_vel[a * B + b] = g[a];
      if (acc) {
        const double u = acc[a * B + b];
        imu_acc[a * B + b] = I.filtered ? I.f[6 * (size_t)b + a].average(u) : u;
      }
    }
    const double w = quat[b], x = quat[B + b], y = quat[2 * B + b], z = quat[3 * B + b];
    double R[9], Z[9], e[3];
    quat_to_rot(w, x, y, z, R);
    quat_to_euler(w, x, y, z, e);
    yaw_to_rot_z(e[2], Z);
    for (int k = 0; k < 9; ++k) { rot[k * B + b] = R[k]; rot_z[k * B + b] = Z[k]; }
    for (int i = 0; i < 3; ++i) {
      euler[i * B + b] = e[i];
      ang_vel[i * B + b] = R[3 * i] * g[0] + R[3 * i + 1] * g[1] + R[3 * i + 2] * g[2];
    }
  }
  return 0;
}

void* oracle_command_new(int B, int variant, double height, double hmin, double hmax, const double* kp3, const double* lock2) {
  Command* c = new Command;
  c->variant = variant;
  c->hmin = hmin; c->hmax = hmax; c->lock[0] = lock2[0]; c->lock[1] = lock2[1];
  c->height.assign(B, height);
  c->euler_d.assign(3 * (size_t)B, 0.0); c->pos_d.assign(3 * (size_t)B, 0.0); c->lin_vel_d.assign(3 * (size_t)B, 0.0);
  c->kp.resize(3 * (size_t)B);
  for (int b = 0; b < B; ++b)
    for (int a = 0; a < 3; ++a) c->kp[3 * (size_t)b + a] = kp3[a];
  c->ctrl.assign(B, 0);
  return c;
}
void oracle_command_free(void* h) { delete static_cast<Command*>(h); }

// one main_update front half for B robots.  cmd [7][B], root_pos [3][B]; euler_d1_in [B] (may be null): root_euler_d[1] as
// compute_grf left it.  Out: movement_mode [B], kp_linear [3][B], ref [9][B] (a1mpc_inputs layout), des [12][B] (stance layout).
int oracle_command(void* h, int B, double dt, const double* cmd, const double* root_pos, const double* euler_d1_in, uint32_t* movement_mode,
                   double* kp_linear, double* ref, double* des) {
  Command& S = *static_cast<Command*>(h);
  const bool hw = S.variant == 1;
  for (int b = 0; b < B; ++b) {
    const double velx = cmd[b], vely = cmd[B + b], velz = cmd[2 * B + b];
    const double roll_rate = cmd[3 * B + b], pitch_rate = cmd[4 * B + b], yaw_rate = cmd[5 * B + b];
    const bool toggle = cmd[6 * B + b] != 0.0;
    double* eul = &S.euler_d[3 * (size_t)b];
    double* pos = &S.pos_d[3 * (size_t)b];
    double* kp = &S.kp[3 * (size_t)b];
    double* lvd = &S.lin_vel_d[3 * (size_t)b];
    if (euler_d1_in) eul[1] = euler_d1_in[b];
    // GazeboA1ROS.cpp:122-130
    double& height = S.height[b];
    height += velz * dt;
    if (height >= S.hmax) height = S.hmax;
    if (height <= S.hmin) height = S.hmin;
    // :140-147
    const int prev = S.ctrl[b];
    if (toggle) S.ctrl[b] = (S.ctrl[b] + 1) % 2;
    const int ctrl = S.ctrl[b];
    // :149-161 (HardwareA1ROS.cpp:121-132, IsaacA1ROS.cpp:99-110): only Gazebo sets root_lin_vel_d[2]
    lvd[0] = velx; lvd[1] = vely;
    if (S.variant == 0) lvd[2] = velz;
    if (hw) {
      eul[0] = roll_rate;
      eul[1] = pitch_rate;
    } else {
      eul[0] += roll_rate * dt;
      eul[1] += pitch_rate * dt;
    }
    eul[2] += yaw_rate * dt;
    pos[2] = height;
    // :163-188
    uint32_t mode;
    if (ctrl == 1) {
      mode = 1;
    } else if (ctrl == 0 && prev == 1) {
      mode = 0;
      pos[0] = root_pos[b]; pos[1] = root_pos[B + b];
      kp[0] = S.lock[0]; kp[1] = S.lock[1];
    } else {
      mode = 0;
    }
    if (mode == 1) {
      if (std::sqrt(lvd[0] * lvd[0] + lvd[1] * lvd[1]) > 0.05) {
        pos[0] = root_pos[b]; pos[1] = root_pos[B + b];
        kp[0] = 0.0; kp[1] = 0.0;
      } else {
        kp[0] = S.lock[0]; kp[1] = S.lock[1];
      }
    }
    movement_mode[b] = mode;
    for (int a = 0; a < 3; ++a) kp_linear[a * B + b] = kp[a];
    const double r[9] = {eul[0], eul[1], roll_rate, pitch_rate, yaw_rate, lvd[0], lvd[1], lvd[2], pos[2]};
    for (int i = 0; i < 9; ++i) ref[i * B + b] = r[i];
    const double d[12] = {eul[0], eul[1], eul[2], pos[0], pos[1], pos[2], lvd[0], lvd[1], lvd[2], roll_rate, pitch_rate, yaw_rate};
    for (int i = 0; i < 12; ++i) des[i * B + b] = d[i];
  }
  return 0;
}

}  // extern "C"
