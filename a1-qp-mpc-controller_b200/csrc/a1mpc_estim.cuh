// a1mpc_estim.cuh -- upstream producers of the path's inputs (SURVEY 8f.4), batched:
//   * leg forward kinematics + Jacobian: A1Kinematics::fk / jac (legKinematics/A1Kinematics.cpp:7-18, bodies :39-131) and the
//     per-tick derived quantities of GazeboA1ROS.cpp:264-279 (foot_vel_rel, foot_pos_abs, foot_vel_abs)
//   * A1BasicEKF::init_state / update_estimation (A1BasicEKF.cpp:56-68, 70-164): 18-state, 28-measurement Kalman filter
// Include from exactly one translation unit (a1mpc_api.cu) -- and from tests/emu (g++, A1MPC_EMU).
#pragma once
#include "a1mpc_device.cuh"

namespace a1mpc {

// -------------------------------------------------------------------------------------------------------------
// Leg kinematics.  The reference evaluates Matlab-generated expansions; in closed form, with q = (hip roll, thigh, calf),
// rho_opt = (cx, cy, cz) the contact offset, rho_fix = (ox, oy, d, lt, lc) body offsets / thigh offset / link lengths,
//   w = cy + d,  h = cz - lc,  M = cx sin(q1+q2) - h cos(q1+q2),  L = lt cos q1 + M
//   p = ( ox + h sin(q1+q2) - lt sin q1 + cx cos(q1+q2),   oy + w cos q0 + L sin q0,   w sin q0 - L cos q0 )
// and J = dp/dq follows by differentiation (column k = d p / d q_k).
// -------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void leg_fk_jac(const double (&q)[3], const double* __restrict__ ro, const double* __restrict__ rf,
                                           double (&p)[3], double (&J)[3][3]) {
  const double s0 = sin(q[0]), c0 = cos(q[0]), s1 = sin(q[1]), c1 = cos(q[1]);
  const double s12 = sin(q[1] + q[2]), c12 = cos(q[1] + q[2]);
  const double cx = ro[0], w = ro[1] + rf[2], hh = ro[2] - rf[4], lt = rf[3];
  const double M = cx * s12 - hh * c12;     // dM/dq1 = dM/dq2 = Rr
  const double Rr = cx * c12 + hh * s12;
  const double L = lt * c1 + M;             // dL/dq1 = Rr - lt s1, dL/dq2 = Rr
  const double Pq = Rr - lt * s1;
  p[0] = rf[0] + hh * s12 - lt * s1 + cx * c12;
  p[1] = rf[1] + w * c0 + L * s0;
  p[2] = w * s0 - L * c0;
  J[0][0] = 0.0;                 J[0][1] = -L;        J[0][2] = -M;
  J[1][0] = -w * s0 + L * c0;    J[1][1] = s0 * Pq;   J[1][2] = s0 * Rr;
  J[2][0] = w * c0 + L * s0;     J[2][1] = -c0 * Pq;  J[2][2] = -c0 * Rr;
}

struct LegParams {
  double rho_opt[12];   // 4 legs x (cx, cy, cz)
  double rho_fix[20];   // 4 legs x (ox, oy, d, lt, lc)
};

// the per-robot body of leg_kinematics_kernel, shared with tick_front_b: keep_abs(k, v) also receives every foot_pos_abs element it stores
template <class KeepAbs>
__device__ __forceinline__ void leg_kinematics_body(int b, size_t ld, const double* __restrict__ joint_pos, const double* __restrict__ joint_vel,
                                                    const double* __restrict__ rot, const LegParams& P, double* __restrict__ foot_pos_rel,
                                                    double* __restrict__ jac, double* __restrict__ foot_vel_rel, double* __restrict__ foot_pos_abs,
                                                    double* __restrict__ foot_vel_abs, KeepAbs&& keep_abs) {
  double R[9];
  if (rot) {
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = rot[(size_t)k * ld + b];
  }
#pragma unroll
  for (int leg = 0; leg < 4; ++leg) {
    double q[3], p[3], J[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a) q[a] = joint_pos[(size_t)(3 * leg + a) * ld + b];
    leg_fk_jac(q, P.rho_opt + 3 * leg, P.rho_fix + 5 * leg, p, J);
    if (foot_pos_rel) {
#pragma unroll
      for (int a = 0; a < 3; ++a) foot_pos_rel[(size_t)(3 * leg + a) * ld + b] = p[a];
    }
    if (jac) {
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) jac[(size_t)(9 * leg + 3 * a + c) * ld + b] = J[a][c];
    }
    double v[3] = {0.0, 0.0, 0.0};
    if (joint_vel) {
      double dq[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) dq[a] = joint_vel[(size_t)(3 * leg + a) * ld + b];
#pragma unroll
      for (int a = 0; a < 3; ++a) v[a] = J[a][0] * dq[0] + J[a][1] * dq[1] + J[a][2] * dq[2];
      if (foot_vel_rel) {
#pragma unroll
        for (int a = 0; a < 3; ++a) foot_vel_rel[(size_t)(3 * leg + a) * ld + b] = v[a];
      }
    }
    if (rot) {
      if (foot_pos_abs) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const double v = R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2];
          foot_pos_abs[(size_t)(3 * leg + a) * ld + b] = v;
          keep_abs(3 * leg + a, v);
        }
      }
      if (foot_vel_abs && joint_vel) {
#pragma unroll
        for (int a = 0; a < 3; ++a) foot_vel_abs[(size_t)(3 * leg + a) * ld + b] = R[3 * a] * v[0] + R[3 * a + 1] * v[1] + R[3 * a + 2] * v[2];
      }
    }
  }
}

// thread per robot; batch-major SoA (ld = B).  Any output pointer may be null.
__global__ void leg_kinematics_kernel(int B, const double* __restrict__ joint_pos, const double* __restrict__ joint_vel,
                                      const double* __restrict__ rot, LegParams P, double* __restrict__ foot_pos_rel,
                                      double* __restrict__ jac, double* __restrict__ foot_vel_rel, double* __restrict__ foot_pos_abs,
                                      double* __restrict__ foot_vel_abs) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  leg_kinematics_body(b, (size_t)B, joint_pos, joint_vel, rot, P, foot_pos_rel, jac, foot_vel_rel, foot_pos_abs, foot_vel_abs, [](int, double) {});
}

#if A1MPC_DMMA
// -------------------------------------------------------------------------------------------------------------
// Kalman filter, one warp per robot.
// Device-resident filter state per robot (a1mpc_ekf_bytes): EKF_STATE_DOUBLES doubles = x[18], P[18][18] row-major.
// The measurement matrix C (A1BasicEKF.cpp:10-17) is never formed: for any 18-vector / 18-row matrix M
//   (C M)[3i+a] = M[6+3i+a] - M[a],  (C M)[12+3i+a] = M[3+a],  (C M)[24+i] = M[6+3i+2]          (i = leg, a = axis)
// The 28x28 innovation covariance S (padded to 32) is factored by the tiled DMMA Cholesky of a1mpc_device.cuh (the
// reference solves with fullPivHouseholderQr, :135/:139 -- S is symmetric positive definite, the solutions agree to
// rounding), and S^-1 [error_y, C Pbar] is 19 right-hand sides solved eight at a time: the rows of the MMA A/C fragment
// that the single-vector solve leaves empty carry seven more vectors for free.
// -------------------------------------------------------------------------------------------------------------
constexpr int EKF_NX = 18, EKF_NY = 28, EKF_NYP = 32;
constexpr int EKF_STATE_DOUBLES = EKF_NX + EKF_NX * EKF_NX;   // 342
constexpr int EKF_LSZ = (EKF_NYP / 8) * (EKF_NYP / 8 + 1) / 2 * 64;   // 640
// per-warp shared memory (doubles)
constexpr int EKF_OFF_X = 0;                        // x (18) + pad
constexpr int EKF_OFF_XB = 20;                      // xbar
constexpr int EKF_OFF_IN = 40;                      // staged inputs: rot 9, acc 3, gyro 3, fk 12, fv 12, force 4, ec 4  (47) + pad
constexpr int EKF_OFF_P = 88;                       // P (324)
constexpr int EKF_OFF_PB = EKF_OFF_P + 324;         // Pbar
constexpr int EKF_OFF_G = EKF_OFF_PB + 324;         // G = C Pbar, 28 x 18
constexpr int EKF_OFF_Y = EKF_OFF_G + 504;          // Y = S^-1 G, 28 x 18
constexpr int EKF_OFF_S = EKF_OFF_Y + 504;          // S tiles (640)
constexpr int EKF_OFF_RB = EKF_OFF_S + EKF_LSZ;     // right-hand-side block 8 x 32
constexpr int EKF_OFF_E = EKF_OFF_RB + 256;         // error_y (32), z = S^-1 error_y (32)
constexpr int EKF_WARP_DOUBLES = EKF_OFF_E + 64;
constexpr int EKF_WPC = 4;

struct EkfParams {
  double dt;
  int assume_flat_ground;
};

// (C v)[r] for an 18-vector v with stride `st`
__device__ __forceinline__ double ekf_crow(const double* v, int st, int r) {
  if (r < 12) { const int a = r % 3; return v[(6 + r) * st] - v[a * st]; }
  if (r < 24) { const int a = (r - 12) % 3; return v[(3 + a) * st]; }
  return v[(6 + 3 * (r - 24) + 2) * st];
}

// eight right-hand sides at once: rb is an 8 x NPAD row-major block (row = right-hand side), solved in place
template <int NPAD>
__device__ __forceinline__ void chol_solve8_impl(const double* __restrict__ L, double* __restrict__ rb, int lane) {
  constexpr int NB = NPAD / 8;
  const int r = lane >> 2, c4 = lane & 3;
  const int orow = tile_pos(r, 2 * c4);
  const int oc0 = tile_pos(2 * c4, r), oc1 = tile_pos(2 * c4 + 1, r);
  d2 acc[NB];
#pragma unroll
  for (int I = 0; I < NB; ++I) acc[I] = ld2(rb + r * NPAD + 8 * I + 2 * c4);
#pragma unroll
  for (int J = 0; J < NB; ++J) {
    const d2 wt = ld2(L + tile_off(J, J) + orow);
    d2 y{0.0, 0.0};
    dmma(y, acc[J].x, wt.x);
    dmma(y, acc[J].y, wt.y);
    acc[J] = y;
    const double nx = -y.x, ny = -y.y;
#pragma unroll
    for (int I = J + 1; I < NB; ++I) {
      const d2 t = ld2(L + tile_off(I, J) + orow);
      dmma(acc[I], nx, t.x);
      dmma(acc[I], ny, t.y);
    }
  }
#pragma unroll
  for (int J = NB - 1; J >= 0; --J) {
    const double* D = L + tile_off(J, J);
    d2 x{0.0, 0.0};
    dmma(x, acc[J].x, D[oc0]);
    dmma(x, acc[J].y, D[oc1]);
    acc[J] = x;
    const double nx = -x.x, ny = -x.y;
#pragma unroll
    for (int I = 0; I < J; ++I) {
      const double* Tl = L + tile_off(J, I);
      dmma(acc[I], nx, Tl[oc0]);
      dmma(acc[I], ny, Tl[oc1]);
    }
  }
#pragma unroll
  for (int I = 0; I < NB; ++I) st2(rb + r * NPAD + 8 * I + 2 * c4, acc[I]);
  __syncwarp();
}

// A1BasicEKF::init_state (A1BasicEKF.cpp:56-68): P = 3 I, x = (0,0,0.09, 0,0,0, R fk_i + pos)
__device__ __forceinline__ void ekf_init_body(int b, int B, double* __restrict__ state, const double* __restrict__ foot_pos_rel,
                                              const double* __restrict__ rot) {
  const size_t ld = (size_t)B;
  double* x = state + (size_t)b * EKF_STATE_DOUBLES;
  double* P = x + EKF_NX;
  for (int i = 0; i < EKF_NX * EKF_NX; ++i) P[i] = 0.0;
  for (int i = 0; i < EKF_NX; ++i) { P[i * EKF_NX + i] = 3.0; x[i] = 0.0; }
  x[2] = 0.09;
  double R[9];
  for (int k = 0; k < 9; ++k) R[k] = rot[(size_t)k * ld + b];
  for (int leg = 0; leg < 4; ++leg) {
    double p[3];
    for (int a = 0; a < 3; ++a) p[a] = foot_pos_rel[(size_t)(3 * leg + a) * ld + b];
    for (int a = 0; a < 3; ++a) x[6 + 3 * leg + a] = R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2] + x[a];
  }
}

__global__ void ekf_init_kernel(int B, double* __restrict__ state, const double* __restrict__ foot_pos_rel, const double* __restrict__ rot) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  ekf_init_body(b, B, state, foot_pos_rel, rot);
}

// A1BasicEKF::update_estimation (A1BasicEKF.cpp:70-164).  Inputs batch-major SoA (ld = B).  status[b] = 0, or 3 when S is
// not positive definite / not finite or error_y is not finite (the state of that robot is then left untouched).
__global__ void __launch_bounds__(32 * EKF_WPC) ekf_update_kernel(int B, EkfParams P, double* __restrict__ state,
                                                                 const uint32_t* __restrict__ movement_mode, const double* __restrict__ imu_acc,
                                                                 const double* __restrict__ imu_ang_vel, const double* __restrict__ rot,
                                                                 const double* __restrict__ foot_pos_rel, const double* __restrict__ foot_vel_rel,
                                                                 const double* __restrict__ foot_force, double* __restrict__ root_pos,
                                                                 double* __restrict__ root_lin_vel, uint32_t* __restrict__ est_contacts,
                                                                 int32_t* __restrict__ status) {
  A1MPC_DYN_SMEM(smem);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  double* ws = smem + wib * EKF_WARP_DOUBLES;
  double* x = ws + EKF_OFF_X; double* xb = ws + EKF_OFF_XB; double* in = ws + EKF_OFF_IN;
  double* Pm = ws + EKF_OFF_P; double* Pb = ws + EKF_OFF_PB; double* G = ws + EKF_OFF_G; double* Y = ws + EKF_OFF_Y;
  double* S = ws + EKF_OFF_S; double* rb = ws + EKF_OFF_RB; double* ev = ws + EKF_OFF_E; double* zv = ev + 32;
  const size_t ld = (size_t)B;
  const double dt = P.dt;
#pragma unroll 1
  for (int b = blockIdx.x * EKF_WPC + wib; b < B; b += gridDim.x * EKF_WPC) {
    double* gx = state + (size_t)b * EKF_STATE_DOUBLES;
    for (int i = lane; i < EKF_NX; i += 32) x[i] = gx[i];
    for (int i = lane; i < EKF_NX * EKF_NX; i += 32) Pm[i] = gx[EKF_NX + i];
    // staged inputs: rot 0..8, acc 9..11, gyro 12..14, fk 15..26, fv 27..38, force 39..42, ec 43..46
    if (lane < 9) in[lane] = rot[(size_t)lane * ld + b];
    if (lane < 3) { in[9 + lane] = imu_acc[(size_t)lane * ld + b]; in[12 + lane] = imu_ang_vel[(size_t)lane * ld + b]; }
    if (lane < 12) { in[15 + lane] = foot_pos_rel[(size_t)lane * ld + b]; in[27 + lane] = foot_vel_rel[(size_t)lane * ld + b]; }
    if (lane < 4) {
      const double ff = foot_force[(size_t)lane * ld + b];
      in[39 + lane] = ff;
      // contact estimation (:78-86): stand -> 1, walk -> clamp(force / 100, 0, 1) with the comparisons of std::max / std::min,
      // so a NaN force stays NaN (fmax / fmin would drop it) and ends the robot NUMERICAL through S
      const double r = ff / (100.0 - 0.0);
      in[43 + lane] = (movement_mode[b] == 0u) ? 1.0 : (r < 0.0 ? 0.0 : (1.0 < r ? 1.0 : r));
    }
    __syncwarp();
    const double* R = in; const double* fk = in + 15; const double* fv = in + 27; const double* ec = in + 43;
    // process update (:111-112): xbar = A x + B u,  u = R a + (0,0,-9.81)
    if (lane < EKF_NX) {
      double v = x[lane];
      if (lane < 3) v += dt * x[3 + lane];
      else if (lane < 6) {
        const int a = lane - 3;
        const double u = R[3 * a] * in[9] + R[3 * a + 1] * in[10] + R[3 * a + 2] * in[11] + (a == 2 ? -9.81 : 0.0);
        v += dt * u;
      }
      xb[lane] = v;
    }
    // Pbar = A P A' + Q with A = I + dt E (E: position rows <- velocity rows), Q diagonal (:88-96)
    for (int e = lane; e < EKF_NX * EKF_NX; e += 32) {
      const int i = e / EKF_NX, j = e - i * EKF_NX;
      double v = Pm[e];
      if (i < 3) v += dt * Pm[(i + 3) * EKF_NX + j];
      if (j < 3) {
        double t = Pm[i * EKF_NX + j + 3];
        if (i < 3) t += dt * Pm[(i + 3) * EKF_NX + j + 3];
        v += dt * t;
      }
      if (i == j) {
        double qd;
        if (i < 3) qd = 0.01 * dt / 20.0;                       // PROCESS_NOISE_PIMU * dt / 20
        else if (i < 6) qd = 0.01 * dt * 9.8 / 20.0;            // PROCESS_NOISE_VIMU * dt * 9.8 / 20
        else qd = (1.0 + (1.0 - ec[(i - 6) / 3]) * 1e3) * dt * 0.01;   // PROCESS_NOISE_PFOOT
        v += qd;
      }
      Pb[e] = v;
    }
    __syncwarp();
    // measurement (:115-130) and its prediction yhat = C xbar: error_y = y - yhat
    if (lane < EKF_NY) {
      double y;
      if (lane < 12) {
        const int i = lane / 3, a = lane - 3 * i;
        y = R[3 * a] * fk[3 * i] + R[3 * a + 1] * fk[3 * i + 1] + R[3 * a + 2] * fk[3 * i + 2];
      } else if (lane < 24) {
        const int i = (lane - 12) / 3, a = lane - 12 - 3 * i;
        const double wx = in[12], wy = in[13], wz = in[14];
        const double px = fk[3 * i], py = fk[3 * i + 1], pz = fk[3 * i + 2];
        // leg_v = -foot_vel_rel - skew(omega) * fk
        const double lv0 = -fv[3 * i] - (wy * pz - wz * py), lv1 = -fv[3 * i + 1] - (wz * px - wx * pz), lv2 = -fv[3 * i + 2] - (wx * py - wy * px);
        const double rl = R[3 * a] * lv0 + R[3 * a + 1] * lv1 + R[3 * a + 2] * lv2;
        y = (1.0 - ec[i]) * x[3 + a] + ec[i] * rl;
      } else {
        const int i = lane - 24;
        y = (1.0 - ec[i]) * (x[2] + fk[3 * i + 2]) + ec[i] * 0.0;
      }
      ev[lane] = y - ekf_crow(xb, 1, lane);
    } else {
      ev[lane] = 0.0;
    }
    // G = C Pbar
    for (int e = lane; e < EKF_NY * EKF_NX; e += 32) {
      const int r = e / EKF_NX, j = e - r * EKF_NX;
      G[e] = ekf_crow(Pb + j, EKF_NX, r);
    }
    __syncwarp();
    // S = 1/2 (G C' + R + transpose) into the tiled factor storage, identity on the padding
    for (int e = lane; e < EKF_NYP * (EKF_NYP + 1) / 2; e += 32) {
      int r = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);
      while (r * (r + 1) / 2 > e) --r;
      while ((r + 1) * (r + 2) / 2 <= e) ++r;
      const int c = e - r * (r + 1) / 2;
      double v;
      if (r >= EKF_NY) v = (r == c) ? 1.0 : 0.0;
      else {
        v = 0.5 * (ekf_crow(G + r * EKF_NX, 1, c) + ekf_crow(G + c * EKF_NX, 1, r));
        if (r == c) {
          double rd;   // sensor noise (:98-108)
          if (r < 12) rd = (1.0 + (1.0 - ec[r / 3]) * 1e3) * 0.001;            // SENSOR_NOISE_PIMU_REL_FOOT
          else if (r < 24) rd = (1.0 + (1.0 - ec[(r - 12) / 3]) * 1e3) * 0.1;  // SENSOR_NOISE_VIMU_REL_FOOT
          else rd = P.assume_flat_ground ? (1.0 + (1.0 - ec[r - 24]) * 1e3) * 0.001 : 1e5;   // SENSOR_NOISE_ZFOOT (:49)
          v += rd;
        }
      }
      S[laddr<EKF_NYP>(r, c)] = v;
    }
    __syncwarp();
    bool ok = chol_inplace_impl<EKF_NYP>(S, lane);
    ok = ok && !__any_sync(0xffffffffu, !(fabs(ev[lane]) < 1e300));
    if (ok) {
      // S^-1 [error_y | G]: 19 right-hand sides in three passes of eight
#pragma unroll 1
      for (int pass = 0; pass < 3; ++pass) {
        for (int e = lane; e < 8 * EKF_NYP; e += 32) {
          const int rr = e / EKF_NYP, k = e - rr * EKF_NYP;
          const int col = 8 * pass + rr - 1;       // -1: error_y
          double v = 0.0;
          if (k < EKF_NY) {
            if (col < 0) v = ev[k];
            else if (col < EKF_NX) v = G[k * EKF_NX + col];
          }
          rb[e] = v;
        }
        __syncwarp();
        chol_solve8_impl<EKF_NYP>(S, rb, lane);
        for (int e = lane; e < 8 * EKF_NYP; e += 32) {
          const int rr = e / EKF_NYP, k = e - rr * EKF_NYP;
          const int col = 8 * pass + rr - 1;
          if (k < EKF_NY) {
            if (col < 0) zv[k] = rb[e];
            else if (col < EKF_NX) Y[k * EKF_NX + col] = rb[e];
          }
        }
        __syncwarp();
      }
      // x = xbar + Pbar C' S^-1 error_y = xbar + G' z (:137)
      if (lane < EKF_NX) {
        double v = xb[lane];
        for (int k = 0; k < EKF_NY; ++k) v = fma(G[k * EKF_NX + lane], zv[k], v);
        x[lane] = v;
      }
      // P = Pbar - G' Y (:140), then 1/2 (P + P') (:141)
      for (int e = lane; e < EKF_NX * EKF_NX; e += 32) {
        const int i = e / EKF_NX, j = e - i * EKF_NX;
        double v = Pb[e];
        for (int k = 0; k < EKF_NY; ++k) v = fma(-G[k * EKF_NX + i], Y[k * EKF_NX + j], v);
        Pm[e] = v;
      }
      __syncwarp();
      for (int e = lane; e < EKF_NX * EKF_NX; e += 32) {
        const int i = e / EKF_NX, j = e - i * EKF_NX;
        Pb[e] = 0.5 * (Pm[e] + Pm[j * EKF_NX + i]);
      }
      __syncwarp();
      // reduce position drift (:144-148)
      const bool cut = (Pb[0] * Pb[EKF_NX + 1] - Pb[1] * Pb[EKF_NX]) > 1e-6;
      for (int e = lane; e < EKF_NX * EKF_NX; e += 32) {
        const int i = e / EKF_NX, j = e - i * EKF_NX;
        double v = Pb[e];
        if (cut) {
          if ((i < 2) != (j < 2)) v = 0.0;
          else if (i < 2 && j < 2) v = v / 10.0;
        }
        gx[EKF_NX + e] = v;
      }
      if (lane < EKF_NX) gx[lane] = x[lane];
    }
    // outputs (:152-163)
    if (lane < 3) {
      if (root_pos) root_pos[(size_t)lane * ld + b] = ok ? x[lane] : gx[lane];
      if (root_lin_vel) root_lin_vel[(size_t)lane * ld + b] = ok ? x[3 + lane] : gx[3 + lane];
    }
    if (lane == 0) {
      if (est_contacts) {
        uint32_t m = 0;
        for (int i = 0; i < 4; ++i) m |= (ec[i] < 0.5 ? 0u : 1u) << i;
        est_contacts[b] = m;
      }
      if (status) status[b] = ok ? A1MPC_STATUS_OPTIMAL : A1MPC_STATUS_NUMERICAL;
    }
    __syncwarp();
  }
}
#endif  // A1MPC_DMMA

}  // namespace a1mpc
