// a1mpc_swing.cuh -- the two control-tick stages between update_plan and the MPC solve, batched, with the controller's own state on
// the device:
//   * A1RobotControl::generate_swing_legs_ctrl (A1RobotControl.cpp:204-287): swing-leg Bezier targets, PD force foot_forces_kin,
//     early-contact detection, contacts = plan | early, recent-contact moving-window filters
//   * the terrain-adaptation front of A1RobotControl::compute_grf (:334-376, compute_walking_surface :566-582): least-squares
//     plane through the four recent-contact points, dihedral angle to flat ground, 100-sample filter, desired pitch
// Include from exactly one translation unit (a1mpc_api.cu) -- and from tests/emu (g++, A1MPC_EMU).
//
// Device-resident state per robot (a1mpc_swing_bytes), batch-major: field f of robot b at state[f * B + b], so the buffer is bound to
// the B it was initialised for.  Fields (doubles):
//   SW_START..  foot_pos_start [12]            SW_RLAST..  foot_pos_rel_last_time [12]   SW_TLAST..  foot_pos_target_last_time [12]
//   SW_RC..     foot_pos_recent_contact [12]   SW_EARLY    early_contacts bit mask
//   SW_FHDR + 4k + {0,1,2,3}: sum, Neumaier correction, fill count, ring head of filter k (k = 3 leg + axis: recent_contact_{x,y,z}
//   _filter[leg]; k = 12: terrain_angle_filter);  SW_FVAL + 60 k + j (k < 12), SW_FVAL + 720 + j (k = 12): window slot j.
// One thread per robot: the per-robot work is a few hundred flops over ~100 doubles of state, the four legs share R_z and the
// early-contact mask, and the terrain stage needs all four legs at once; batch-major fields keep every load and store coalesced.
#pragma once
#include "a1mpc_device.cuh"
#include "a1mpc_filter.cuh"

namespace a1mpc {

constexpr int SW_RC_WINDOW = 60;       // recent_contact_{x,y,z}_filter (A1RobotControl.cpp:53-57)
constexpr int SW_TA_WINDOW = 100;      // terrain_angle_filter (:52)
constexpr int SW_START = 0, SW_RLAST = 12, SW_TLAST = 24, SW_RC = 36, SW_EARLY = 48;
constexpr int SW_FHDR = 49;
constexpr int SW_FVAL = SW_FHDR + 13 * 4;
constexpr int SW_FIELDS = SW_FVAL + 12 * SW_RC_WINDOW + SW_TA_WINDOW;   // 921 doubles per robot
constexpr double SW_FOOT_FORCE_LOW = 30.0;                              // FOOT_FORCE_LOW (A1Params.h:38)
constexpr double SW_CLEARANCE1 = (double)0.0f, SW_CLEARANCE2 = (double)0.4f;   // float literals (A1Params.h:41-42)

struct SwingParams {
  double cps, dt;      // counter_per_swing, control period
  double kp[12], kd[12];   // kp_foot, kd_foot leg-major: [3 leg + axis]
};

// filter k of the robot whose swing state starts at s (stride ld)
__device__ __forceinline__ double sw_filter(double* s, size_t ld, int k, double x) {
  return mw_filter(s, ld, k < 12 ? SW_RC_WINDOW : SW_TA_WINDOW, SW_FVAL + SW_RC_WINDOW * k, SW_FHDR + 4 * k, x);
}

// BezierUtils::bezier_curve (utils/Utils.cpp:100-107), degree 4: sum_i C(4,i) t^i (1-t)^(4-i) P_i accumulated in index order.  The
// powers are products (t^2 is exact for a float t, t^3 and t^4 are rounded once).
__device__ __forceinline__ double sw_bezier(double t, const double (&P)[5]) {
  const double u = 1.0 - t, t2 = t * t, u2 = u * u;
  const double tp[5] = {1.0, t, t2, t2 * t, t2 * t2};
  const double up[5] = {1.0, u, u2, u2 * u, u2 * u2};
  const double c[5] = {1.0, 4.0, 6.0, 4.0, 1.0};
  double y = 0.0;
#pragma unroll
  for (int i = 0; i < 5; ++i) y += c[i] * tp[i] * up[4 - i] * P[i];
  return y;
}

// zero state = A1CtrlStates::reset() values of the fields above (A1CtrlStates.h:83-100) and fresh filters (A1RobotControl.cpp:52-57)
__device__ __forceinline__ void swing_init_body(int b, int B, double* __restrict__ state) {
  for (int f = 0; f < SW_FIELDS; ++f) state[(size_t)f * B + b] = 0.0;
}

__global__ void swing_init_kernel(int B, double* __restrict__ state) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  swing_init_body(b, B, state);
}

// one leg of generate_swing_legs_ctrl (A1RobotControl.cpp:204-287) for the robot whose swing state starts at s.  src gives the stage's
// per-robot inputs: plan(), g(i) = gait_counter, p(i, a) = foot_pos_abs, fin(i, a) = foot_pos_target_rel.
template <class Src>
__device__ __forceinline__ void swing_leg(int i, int b, size_t ld, const SwingParams& P, double* __restrict__ s, const double (&R)[9], uint32_t pm,
                                          uint32_t& early, uint32_t& cm, const Src& src, const double* __restrict__ ff, double* __restrict__ fkin,
                                          double* __restrict__ cur_out, double* __restrict__ rc_out) {
  double p[3], cur[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) p[a] = src.p(i, a);
#pragma unroll
  for (int a = 0; a < 3; ++a) cur[a] = R[a] * p[0] + R[3 + a] * p[1] + R[6 + a] * p[2];   // R_z^T p  (:224)
  const double g = src.g(i);
  float t = 0.0f;
  double st[3];
  if (g <= P.cps) {   // stance: keep refreshing foot_pos_start (:227-232)
#pragma unroll
    for (int a = 0; a < 3; ++a) { st[a] = cur[a]; s[(size_t)(SW_START + 3 * i + a) * ld] = cur[a]; }
  } else {            // swing: spline time in single precision (:235)
    t = (float)(g - P.cps) / (float)P.cps;
#pragma unroll
    for (int a = 0; a < 3; ++a) st[a] = s[(size_t)(SW_START + 3 * i + a) * ld];
  }
  // BezierUtils::get_foot_pos_curve with terrain pitch literal 0.0 (:238-241, Utils.cpp:64-97)
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
  // finite-difference velocities against the stored last positions, PD force (:243-252)
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
  // early contact (:259-267): sticky, cleared only when gc <= 1.5 cps
  const bool planned = (pm >> i) & 1u;
  if (g <= P.cps * 1.5) early &= ~(1u << i);
  if (!planned && g > P.cps * 1.5 && ff[(size_t)i * ld + b] > SW_FOOT_FORCE_LOW) early |= 1u << i;
  const bool c = planned || ((early >> i) & 1u);
  if (c) {   // (:271-281) the leg's three recent-contact filters move on contact ticks only
    cm |= 1u << i;
#pragma unroll
    for (int a = 0; a < 3; ++a) s[(size_t)(SW_RC + 3 * i + a) * ld] = sw_filter(s, ld, 3 * i + a, p[a]);
  }
  if (rc_out) {
#pragma unroll
    for (int a = 0; a < 3; ++a) rc_out[(size_t)(3 * i + a) * ld + b] = s[(size_t)(SW_RC + 3 * i + a) * ld];
  }
}

// the per-robot body of swing_legs_kernel (tick_front_b runs the same rolled loop of swing_leg, each leg after its foothold target)
template <class Src>
__device__ __forceinline__ void swing_legs_body(int b, size_t ld, const SwingParams& P, double* __restrict__ state, const Src& src,
                                                const double* __restrict__ rz, const double* __restrict__ ff, double* __restrict__ fkin,
                                                uint32_t* __restrict__ contacts, double* __restrict__ cur_out, double* __restrict__ rc_out) {
  double* s = state + b;
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = rz[(size_t)k * ld + b];
  const uint32_t pm = src.plan();
  uint32_t early = (uint32_t)s[(size_t)SW_EARLY * ld];
  uint32_t cm = 0;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) swing_leg(i, b, ld, P, s, R, pm, early, cm, src, ff, fkin, cur_out, rc_out);
  s[(size_t)SW_EARLY * ld] = (double)early;
  contacts[b] = cm;
}

// the inputs of swing_legs_kernel: batch-major arrays
struct SwingSrcArrays {
  const double* gc;
  const uint32_t* pl;
  const double* fpa;
  const double* tgt;
  size_t ld;
  int b;
  __device__ __forceinline__ uint32_t plan() const { return pl[b]; }
  __device__ __forceinline__ double g(int i) const { return gc[(size_t)i * ld + b]; }
  __device__ __forceinline__ double p(int i, int a) const { return fpa[(size_t)(3 * i + a) * ld + b]; }
  __device__ __forceinline__ double fin(int i, int a) const { return tgt[(size_t)(3 * i + a) * ld + b]; }
};

// generate_swing_legs_ctrl (A1RobotControl.cpp:204-287), thread per robot.  cur_out / rc_out may be null.
__global__ void swing_legs_kernel(int B, SwingParams P, double* __restrict__ state, const double* __restrict__ gc,
                                  const uint32_t* __restrict__ plan, const double* __restrict__ rz, const double* __restrict__ fpa,
                                  const double* __restrict__ tgt, const double* __restrict__ ff, double* __restrict__ fkin,
                                  uint32_t* __restrict__ contacts, double* __restrict__ cur_out, double* __restrict__ rc_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  const SwingSrcArrays src{gc, plan, fpa, tgt, ld, b};
  swing_legs_body(b, ld, P, state, src, rz, ff, fkin, contacts, cur_out, rc_out);
}

// Utils::pseudo_inverse of the symmetric positive semidefinite 3x3 A (utils/Utils.cpp:44-52) applied to v: the singular values of A
// are the moduli of its eigenvalues, so cyclic Jacobi sweeps give A = V diag(l) V^T and pinv(A) v = sum over |l_k| > eps 3 max|l|
// of V_k (V_k . v) / l_k -- the reference's cutoff.
__device__ __forceinline__ void sw_pinv_apply(double (&A)[3][3], const double (&v)[3], double (&x)[3]) {
  double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
#pragma unroll 1
  for (int sweep = 0; sweep < 12; ++sweep) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    const double dg = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (!(off > 1e-40 * dg)) break;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2, r = 3 - p - q;
      const double apq = A[p][q];
      if (apq == 0.0) continue;
      const double th = (A[q][q] - A[p][p]) / (2.0 * apq);
      const double t = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
      A[p][p] -= t * apq;
      A[q][q] += t * apq;
      A[p][q] = A[q][p] = 0.0;
      const double arp = A[r][p], arq = A[r][q];
      A[r][p] = A[p][r] = c * arp - sn * arq;
      A[r][q] = A[q][r] = sn * arp + c * arq;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double vp = V[k][p], vq = V[k][q];
        V[k][p] = c * vp - sn * vq;
        V[k][q] = sn * vp + c * vq;
      }
    }
  }
  const double lmax = fmax(fabs(A[0][0]), fmax(fabs(A[1][1]), fabs(A[2][2])));
  const double tol = 2.220446049250313e-16 * 3.0 * lmax;   // numeric_limits<double>::epsilon() * max(rows, cols) * sigma_max
  x[0] = x[1] = x[2] = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (!(fabs(A[k][k]) > tol)) continue;
    const double w = (V[0][k] * v[0] + V[1][k] * v[1] + V[2][k] * v[2]) / A[k][k];
#pragma unroll
    for (int a = 0; a < 3; ++a) x[a] += V[a][k] * w;
  }
}

// the least-squares plane z = a0 + a1 x + a2 y through the four recent-contact points of the robot whose swing state starts at s
// (compute_walking_surface, A1RobotControl.cpp:566-582): the fit of terrain_body, term for term.  terrain_body keeps its own copy
// because handing the plane out of it changes the code the compiler makes of terrain_pitch_kernel.
__device__ __forceinline__ void sw_plane(const double* s, size_t ld, double (&a)[3]) {
  double x[4], y[4], z[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[i] = s[(size_t)(SW_RC + 3 * i) * ld];
    y[i] = s[(size_t)(SW_RC + 3 * i + 1) * ld];
    z[i] = s[(size_t)(SW_RC + 3 * i + 2) * ld];
  }
  // W = [1 x y] (4 x 3): W^T W and W^T z
  double A[3][3], v[3] = {0.0, 0.0, 0.0};
  double sx = 0.0, sy = 0.0, sxx = 0.0, sxy = 0.0, syy = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sx += x[i]; sy += y[i]; sxx += x[i] * x[i]; sxy += x[i] * y[i]; syy += y[i] * y[i];
    v[0] += z[i]; v[1] += x[i] * z[i]; v[2] += y[i] * z[i];
  }
  A[0][0] = 4.0; A[0][1] = A[1][0] = sx; A[0][2] = A[2][0] = sy;
  A[1][1] = sxx; A[1][2] = A[2][1] = sxy; A[2][2] = syy;
  sw_pinv_apply(A, v, a);
}

// the per-robot body of terrain_pitch_kernel: terrain adaptation of compute_grf (A1RobotControl.cpp:334-376).  ref row 1
// (root_euler_d[1]) is written only when adapt != 0; pitch (may be null) always.
__device__ __forceinline__ void terrain_body(int b, int B, double* __restrict__ state, int adapt, const double* __restrict__ root_pos,
                                             double* __restrict__ ref, size_t ref_ld, double* __restrict__ pitch) {
  const size_t ld = (size_t)B;
  double* s = state + b;
  double x[4], y[4], z[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[i] = s[(size_t)(SW_RC + 3 * i) * ld];
    y[i] = s[(size_t)(SW_RC + 3 * i + 1) * ld];
    z[i] = s[(size_t)(SW_RC + 3 * i + 2) * ld];
  }
  // W = [1 x y] (4 x 3): W^T W and W^T z
  double A[3][3], v[3] = {0.0, 0.0, 0.0};
  double sx = 0.0, sy = 0.0, sxx = 0.0, sxy = 0.0, syy = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sx += x[i]; sy += y[i]; sxx += x[i] * x[i]; sxy += x[i] * y[i]; syy += y[i] * y[i];
    v[0] += z[i]; v[1] += x[i] * z[i]; v[2] += y[i] * z[i];
  }
  A[0][0] = 4.0; A[0][1] = A[1][0] = sx; A[0][2] = A[2][0] = sy;
  A[1][1] = sxx; A[1][2] = A[2][1] = sxy; A[2][2] = syy;
  double a[3];
  sw_pinv_apply(A, v, a);
  // surface a1 x + a2 y - z + a0 = 0 against flat ground (0, 0, 1): |(-1)| / (1 * |(a1, a2, -1)|)
  const double ang = acos(1.0 / sqrt(a[1] * a[1] + a[2] * a[2] + 1.0));
  double angle = 0.0;
  if (root_pos[2 * ld + b] > 0.1) angle = sw_filter(s, ld, 12, ang);   // only record the angle when the body is high (:341-345)
  if (angle > 0.5) angle = 0.5;
  if (angle < -0.5) angle = -0.5;
  const double fr = z[0] + z[1] - z[2] - z[3];   // F_R_diff (:355-356)
  if (adapt) ref[ref_ld + b] = fr > 0.05 ? -angle : angle;
  if (pitch) pitch[b] = angle;
}

// terrain adaptation of compute_grf, thread per robot
__global__ void terrain_pitch_kernel(int B, double* __restrict__ state, int adapt, const double* __restrict__ root_pos,
                                     double* __restrict__ ref, size_t ref_ld, double* __restrict__ pitch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  terrain_body(b, B, state, adapt, root_pos, ref, ref_ld, pitch);
}

constexpr double SW_TILT_MAX = 0.5;                                                   // the angle clip of A1RobotControl.cpp:347-352
constexpr double SW_TILT_SIN = 0.479425538604203, SW_TILT_COS = 0.8775825618903728;   // sin 0.5, cos 0.5

// the walking surface's unit normal in the world frame from the swing state of the robot that starts at s and its root_pos z: the
// fitted plane's own normal (-a1, -a2, 1) / |.|, its tilt clipped to 0.5 rad about the same horizontal axis, e_z while z <= 0.1
__device__ __forceinline__ void sw_surface_normal(const double* s, size_t ld, double root_z, double (&n)[3]) {
  double a[3];
  sw_plane(s, ld, a);
  n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
  if (root_z > 0.1) {
    if (acos(1.0 / sqrt(a[1] * a[1] + a[2] * a[2] + 1.0)) > SW_TILT_MAX) {   // terrain_body's angle before the filter
      const double h = SW_TILT_SIN / sqrt(a[1] * a[1] + a[2] * a[2]);
      n[0] = -a[1] * h; n[1] = -a[2] * h; n[2] = SW_TILT_COS;
    } else {
      const double inv = 1.0 / sqrt(a[1] * a[1] + a[2] * a[2] + 1.0);
      n[0] = -a[1] * inv; n[1] = -a[2] * inv; n[2] = inv;
    }
  }
}

// terrain_pitch_kernel's stage, and the walking surface's unit normal in the world frame for the friction pyramids of the solve:
// normals [12][B], the same for all four feet.  The plane is fitted in the frame of foot_pos_recent_contact (world axes), so its normal
// is (-a1, -a2, 1) / |.|; a tilt beyond 0.5 rad is clipped to 0.5 about the same horizontal axis, and while the body is low (the filter
// records nothing) the normal is e_z.  n_z >= cos 0.5 > 0 always.  sched (may be null): the held pattern, contacts [B] copied into all
// N rows.  The plane is fitted again after the stage, which does not write the recent-contact points (sw_plane).
__global__ void terrain_normals_kernel(int B, double* __restrict__ state, int adapt, const double* __restrict__ root_pos,
                                       double* __restrict__ ref, size_t ref_ld, double* __restrict__ pitch, double* __restrict__ normals,
                                       const uint32_t* __restrict__ contacts, uint32_t* __restrict__ sched, int N) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  terrain_body(b, B, state, adapt, root_pos, ref, ref_ld, pitch);
  double n[3];
  sw_surface_normal(state + b, ld, root_pos[2 * ld + b], n);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) normals[(size_t)(3 * i + k) * ld + b] = n[k];
  if (sched) {
    const uint32_t c = contacts[b];
    for (int k = 0; k < N; ++k) sched[(size_t)k * ld + b] = c;
  }
}

// the walking surface's normal of terrain_normals_kernel without the terrain stage, thread per robot: the ESTIMATED source of a QP-mode tick
// (the reference adapts to terrain only in MPC mode, so terrain_angle_filter and ref stay as they are).  It only reads the swing state,
// whose recent-contact points the swing stage records in both modes; normals [12][B], the same for all four feet.
__global__ void surface_normals_kernel(int B, const double* __restrict__ state, const double* __restrict__ root_pos, double* __restrict__ normals) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const size_t ld = (size_t)B;
  double n[3];
  sw_surface_normal(state + b, ld, root_pos[2 * ld + b], n);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) normals[(size_t)(3 * i + k) * ld + b] = n[k];
}

}  // namespace a1mpc
