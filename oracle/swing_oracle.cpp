// oracle/swing_oracle.cpp -- TEST INFRASTRUCTURE, not product code: the oracle of a1mpc_swing_legs_batch / a1mpc_terrain_pitch_batch.
// Built by `make -C oracle -f swing.mk` into oracle/liba1mpc_swing_oracle.so, bound by oracle/swing_oracle_py.py.  Nothing under
// a1-qp-mpc-controller_b200/ may include, link or call this file.  Dependency-free C++17.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <limits>
#include <vector>

// ---------------------------------------------------------------------------------------------------------------------
// Swing-leg control and terrain pitch: A1RobotControl::generate_swing_legs_ctrl (A1RobotControl.cpp:204-287) and the terrain front of
// compute_grf (:334-376, compute_walking_surface :566-582), restated per robot with the controller's state in a plain struct and the
// moving-window filters (utils/filter.hpp) as std::deque windows.  The Bezier powers are std::pow as in the reference; the
// least-squares plane is solved through a long-double Jacobi eigen-decomposition of W^T W with the reference's pseudo-inverse cutoff
// (eps * 3 * sigma_max).  PINNED to the reference build by tests/test_swing_ref_pin.py (tests/golden/swing_v1.npz).
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct OracleWindow {
  size_t n;
  std::deque<double> q;
  double sum = 0.0, corr = 0.0;
  explicit OracleWindow(size_t n_) : n(n_) {}
  void add(double v) {   // Neumaier's compensated sum, branch on |sum| >= |v|
    const double t = sum + v;
    if (std::fabs(sum) >= std::fabs(v)) corr += (sum - t) + v;
    else corr += (v - t) + sum;
    sum = t;
  }
  double average(double v) {
    if (q.size() >= n) { add(-q.front()); q.pop_front(); }
    add(v);
    q.push_back(v);
    return (sum + corr) / double(n);   // the full window size, also while filling
  }
};
struct OracleSwing {
  double start[12] = {}, rlast[12] = {}, tlast[12] = {}, recent[12] = {};
  bool early[4] = {false, false, false, false};
  std::vector<OracleWindow> rc = std::vector<OracleWindow>(12, OracleWindow(60));
  OracleWindow terrain = OracleWindow(100);
};
double oracle_bezier4(double t, const double* P) {
  static const double coef[5] = {1, 4, 6, 4, 1};
  const float degree = 4;
  double y = 0;
  for (int i = 0; i <= 4; ++i) y += coef[i] * std::pow(t, i) * std::pow(1 - t, degree - i) * P[i];
  return y;
}
// a = pinv(W^T W) W^T z for W = [1 x y] over the four recent-contact points
void oracle_walking_surface(const double* recent, double* a) {
  typedef long double LD;
  LD M[3][3] = {}, v[3] = {};
  for (int i = 0; i < 4; ++i) {
    const LD w[3] = {1.0L, recent[3 * i], recent[3 * i + 1]};
    for (int r = 0; r < 3; ++r) {
      v[r] += w[r] * (LD)recent[3 * i + 2];
      for (int c = 0; c < 3; ++c) M[r][c] += w[r] * w[c];
    }
  }
  LD V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 50; ++sweep) {
    LD off = 0;
    for (int r = 0; r < 3; ++r) for (int c = r + 1; c < 3; ++c) off += M[r][c] * M[r][c];
    if (off == 0) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (M[p][q] == 0) continue;
        const LD th = (M[q][q] - M[p][p]) / (2 * M[p][q]);
        const LD t = (th >= 0 ? 1 : -1) / (std::fabs(th) + std::sqrt(th * th + 1));
        const LD c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 3; ++k) {   // columns p, q of M J
          const LD mp = M[k][p], mq = M[k][q];
          M[k][p] = c * mp - s * mq; M[k][q] = s * mp + c * mq;
        }
        for (int k = 0; k < 3; ++k) {   // rows p, q of J^T (M J)
          const LD mp = M[p][k], mq = M[q][k];
          M[p][k] = c * mp - s * mq; M[q][k] = s * mp + c * mq;
        }
        M[p][q] = M[q][p] = 0;
        for (int k = 0; k < 3; ++k) {
          const LD vp = V[k][p], vq = V[k][q];
          V[k][p] = c * vp - s * vq; V[k][q] = s * vp + c * vq;
        }
      }
  }
  double smax = 0;
  for (int k = 0; k < 3; ++k) smax = std::max(smax, (double)std::fabs(M[k][k]));
  const double tol = std::numeric_limits<double>::epsilon() * 3 * smax;
  LD x[3] = {0, 0, 0};
  for (int k = 0; k < 3; ++k) {
    if (!((double)std::fabs(M[k][k]) > tol)) continue;
    const LD w = (V[0][k] * v[0] + V[1][k] * v[1] + V[2][k] * v[2]) / M[k][k];
    for (int r = 0; r < 3; ++r) x[r] += V[r][k] * w;
  }
  for (int r = 0; r < 3; ++r) a[r] = (double)x[r];
}
}  // namespace

extern "C" {

void* oracle_swing_new(int B) { return new std::vector<OracleSwing>((size_t)(B > 0 ? B : 0)); }
void oracle_swing_free(void* h) { delete static_cast<std::vector<OracleSwing>*>(h); }

// one generate_swing_legs_ctrl tick for B robots; batch-major SoA (ld = B) as a1mpc_swing_legs_batch; cur / recent may be null
int oracle_swing_legs(void* h, int B, double cps, double dt, const double* kp, const double* kd, const double* gc, const uint32_t* plan,
                      const double* rot_z, const double* foot_abs, const double* target_rel, const double* foot_force, double* f_kin,
                      uint32_t* contacts, double* cur_out, double* recent_out) {
  std::vector<OracleSwing>& S = *static_cast<std::vector<OracleSwing>*>(h);
  if ((int)S.size() != B) return 1;
  const size_t ld = (size_t)B;
  for (int b = 0; b < B; ++b) {
    OracleSwing& s = S[(size_t)b];
    uint32_t m = 0;
    for (int i = 0; i < 4; ++i) {
      double p[3], cur[3], fin[3], tgt[3];
      for (int a = 0; a < 3; ++a) { p[a] = foot_abs[(size_t)(3 * i + a) * ld + b]; fin[a] = target_rel[(size_t)(3 * i + a) * ld + b]; }
      for (int a = 0; a < 3; ++a) {   // root_rot_mat_z^T p
        cur[a] = 0;
        for (int k = 0; k < 3; ++k) cur[a] += rot_z[(size_t)(3 * k + a) * ld + b] * p[k];
      }
      const double g = gc[(size_t)i * ld + b];
      float t;
      if (g <= cps) { t = 0.0; for (int a = 0; a < 3; ++a) s.start[3 * i + a] = cur[a]; }
      else t = float(g - cps) / float(cps);
      const double X[5] = {s.start[3 * i], s.start[3 * i], fin[0], fin[0], fin[0]};
      const double Y[5] = {s.start[3 * i + 1], s.start[3 * i + 1], fin[1], fin[1], fin[1]};
      double Z[5] = {s.start[3 * i + 2], s.start[3 * i + 2], fin[2], fin[2], fin[2]};
      Z[1] += 0.0f;                            // FOOT_SWING_CLEARANCE1
      Z[2] += 0.4f + 0.5 * std::sin(0.0);      // FOOT_SWING_CLEARANCE2, terrain pitch literal 0.0
      tgt[0] = oracle_bezier4(t, X); tgt[1] = oracle_bezier4(t, Y); tgt[2] = oracle_bezier4(t, Z);
      for (int a = 0; a < 3; ++a) {
        const int k = 3 * i + a;
        const double vc = (cur[a] - s.rlast[k]) / dt, vt = (tgt[a] - s.tlast[k]) / dt;
        s.rlast[k] = cur[a];
        s.tlast[k] = tgt[a];
        f_kin[(size_t)k * ld + b] = (tgt[a] - cur[a]) * kp[k] + (vt - vc) * kd[k];
        if (cur_out) cur_out[(size_t)k * ld + b] = cur[a];
      }
      const bool pl = (plan[b] >> i) & 1u;
      if (g <= cps * 1.5) s.early[i] = false;
      if (!pl && g > cps * 1.5 && foot_force[(size_t)i * ld + b] > 30.0) s.early[i] = true;
      if (pl || s.early[i]) {
        m |= 1u << i;
        for (int a = 0; a < 3; ++a) s.recent[3 * i + a] = s.rc[(size_t)(3 * i + a)].average(p[a]);
      }
      if (recent_out) for (int a = 0; a < 3; ++a) recent_out[(size_t)(3 * i + a) * ld + b] = s.recent[3 * i + a];
    }
    contacts[b] = m;
  }
  return 0;
}

// compute_grf's terrain adaptation for B robots: root_pos [3][B]; ref row 1 (ld ref_ld) written when adapt; pitch [B] may be null
int oracle_terrain_pitch(void* h, int B, int adapt, const double* root_pos, double* ref, size_t ref_ld, double* pitch) {
  std::vector<OracleSwing>& S = *static_cast<std::vector<OracleSwing>*>(h);
  if ((int)S.size() != B) return 1;
  for (int b = 0; b < B; ++b) {
    OracleSwing& s = S[(size_t)b];
    double a[3];
    oracle_walking_surface(s.recent, a);
    const double sc[3] = {a[1], a[2], -1.0}, fl[3] = {0.0, 0.0, 1.0};
    const double cosang = std::fabs(fl[0] * sc[0] + fl[1] * sc[1] + fl[2] * sc[2]) /
                          (std::sqrt(fl[0] * fl[0] + fl[1] * fl[1] + fl[2] * fl[2]) * std::sqrt(sc[0] * sc[0] + sc[1] * sc[1] + sc[2] * sc[2]));
    double angle = 0.0;
    if (root_pos[2 * (size_t)B + b] > 0.1) angle = s.terrain.average(std::acos(cosang));
    if (angle > 0.5) angle = 0.5;
    if (angle < -0.5) angle = -0.5;
    const double fr = s.recent[2] + s.recent[5] - s.recent[8] - s.recent[11];
    if (adapt) ref[ref_ld + b] = fr > 0.05 ? -angle : angle;
    if (pitch) pitch[b] = angle;
  }
  return 0;
}

}  // extern "C"
