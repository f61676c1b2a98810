// a1mpc_dense.cu -- QP-major side entry points:
//   * ConvexMpc::calculate_qp_mats for caller-supplied A_d / B_mat_d_list (ConvexMpc.cpp:158-217;
//     the public API lets B_d differ per step, test/test_mpc.cpp:106-122)
//   * OsqpEigen::Solver replacement on a dense Hessian (A1RobotControl.cpp:522-555)
//   * compute_grf's single-step QP branch (A1RobotControl.cpp:11-48, 377-445), on caller-computed root_acc (QP-major) or
//     from the controller state with the PD law in front of it (batch-major)
// All three reuse the interior-point + finisher core of a1mpc_device.cuh through DenseHess.
#ifndef A1MPC_EMU
#include "a1mpc_internal.h"
#else
#include "a1mpc_device.cuh"   // tests/emu/ compiles the kernels of this file with g++ (test infrastructure)
#endif

namespace a1mpc {

// ------------------------------------------------------------------------------------------------
// general rollout + dense Hessian/gradient, one CTA per QP.  For step i the row block
// W_j = A_d^{i-j} B_j (j <= i) is built in shared memory and its contribution W_j1' Q W_j2 is
// accumulated into H (first touch of a block happens at i = max(j1,j2), so H needs no zero fill).
// ------------------------------------------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(256) qp_mats_kernel(const __grid_constant__ DevParams P, int B, const double* __restrict__ A_d,
                                                      const double* __restrict__ B_list, const double* __restrict__ x0,
                                                      const double* __restrict__ x_d, double* __restrict__ H, double* __restrict__ g,
                                                      double* __restrict__ Aqp, double* __restrict__ Bqp) {
  A1MPC_DYN_SMEM(sm);
  double* Apow = sm;                 // N x 169 : A_d^{k+1}
  double* W = Apow + N * 169;        // N x 13 x 12 : row block i of B_qp
  double* qe = W + N * 156;          // 13
  double* xs = qe + 13;              // 13 : A_d^{i+1} x0
  const int b = blockIdx.x;
  if (b >= B) return;
  const int tid = threadIdx.x;
  constexpr int n = 12 * N;
  const double* Ad = A_d + (size_t)b * 169;
  const double* Bl = B_list + (size_t)b * 13 * N * 12;
  double* Hb = H ? H + (size_t)b * n * n : nullptr;
  double* gb = g ? g + (size_t)b * n : nullptr;
  // optional: the public ConvexMpc members A_qp [13N x 13] and B_qp [13N x 12N] (ConvexMpc.h:77-78), row-major, QP-major
  double* Aq = Aqp ? Aqp + (size_t)b * 13 * N * 13 : nullptr;
  double* Bq = Bqp ? Bqp + (size_t)b * 13 * N * n : nullptr;
  for (int e = tid; e < 169; e += blockDim.x) Apow[e] = Ad[e];
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    // A_qp block i (ConvexMpc.cpp:185-191): A_qp[i] = A_qp[i-1] * A_d
    if (i > 0) {
      for (int e = tid; e < 169; e += blockDim.x) {
        const int r = e / 13, c = e - 13 * r;
        double s = 0.0;
        for (int k = 0; k < 13; ++k) s = fma(Apow[(i - 1) * 169 + r * 13 + k], Ad[k * 13 + c], s);
        Apow[i * 169 + e] = s;
      }
    }
    __syncthreads();
    // B_qp row block i (:192-201) and the weighted free-response error (:215-216)
    for (int e = tid; e < (i + 1) * 156; e += blockDim.x) {
      const int j = e / 156, rc = e - 156 * j, r = rc / 12, c = rc - 12 * r;
      double s;
      if (i == j) s = Bl[(size_t)(13 * j + r) * 12 + c];
      else {
        s = 0.0;
        const double* Ap = Apow + (i - j - 1) * 169 + r * 13;
        for (int k = 0; k < 13; ++k) s = fma(Ap[k], Bl[(size_t)(13 * j + k) * 12 + c], s);
      }
      W[e] = s;
    }
    if (tid < 13) {
      double s = 0.0;
      for (int k = 0; k < 13; ++k) s = fma(Apow[i * 169 + tid * 13 + k], x0[(size_t)b * 13 + k], s);
      qe[tid] = (s - x_d[(size_t)b * 13 * N + 13 * i + tid]) * P.q2[tid];
    }
    __syncthreads();
    if (Aq)
      for (int e = tid; e < 169; e += blockDim.x) Aq[(size_t)i * 169 + e] = Apow[i * 169 + e];
    if (Bq)
      for (int e = tid; e < 13 * n; e += blockDim.x) {   // row block i: W for the block columns j <= i, zero to the right (:70-108 reset)
        const int r = e / n, cc = e - n * r, j = cc / 12, c = cc - 12 * j;
        Bq[(size_t)(13 * i + r) * n + cc] = (j <= i) ? W[j * 156 + r * 12 + c] : 0.0;
      }
    const int ni = 12 * (i + 1);
    if (Hb)
    for (int e = tid; e < ni * ni; e += blockDim.x) {
      const int r = e / ni, c = e - ni * r;
      const int j1 = r / 12, a = r - 12 * j1, j2 = c / 12, bb = c - 12 * j2;
      const double* w1 = W + j1 * 156 + a;
      const double* w2 = W + j2 * 156 + bb;
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 13; ++k) s = fma(w1[12 * k] * P.q2[k], w2[12 * k], s);
      const int mx = j1 > j2 ? j1 : j2;
      double* dst = Hb + (size_t)r * n + c;
      if (mx == i) *dst = s + ((r == c) ? P.r2[a] : 0.0);
      else *dst += s;
    }
    if (gb)
    for (int r = tid; r < ni; r += blockDim.x) {
      const int j1 = r / 12, a = r - 12 * j1;
      const double* w1 = W + j1 * 156 + a;
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 13; ++k) s = fma(w1[12 * k], qe[k], s);
      if (j1 == i) gb[r] = s;
      else gb[r] += s;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// classify QPs by the number of stance feet (QP-major APIs)
// ------------------------------------------------------------------------------------------------
__global__ void classify_kernel(int B, const uint32_t* __restrict__ contact, int* __restrict__ list, int* __restrict__ count,
                                double* __restrict__ out, int out_per_qp, int32_t* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int ns = __popc(contact[b] & 15u);
  if (ns == 0) {
    for (int k = 0; k < out_per_qp; ++k) out[(size_t)b * out_per_qp + k] = 0.0;
    status[b] = A1MPC_STATUS_NO_CONTACT;
    return;
  }
  const int slot = atomicAdd(&count[ns], 1);
  list[(size_t)(ns - 1) * B + slot] = b;
}

__global__ void mark_unsupported_kernel(const int* __restrict__ list, const int* __restrict__ count, int cls, double* __restrict__ out,
                                        int out_per_qp, int32_t* __restrict__ status) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= count[cls]) return;
  const int b = list[q];
  for (int k = 0; k < out_per_qp; ++k) out[(size_t)b * out_per_qp + k] = 0.0;
  status[b] = A1MPC_STATUS_NUMERICAL;
}

template <int NS, int N>
struct DenseGeo {
  using G = Geo<NS, N>;
  static constexpr int HS = ((G::NV * G::NV + 1) / 2) * 2;
  static constexpr int WARP_DOUBLES = G::WARP_DOUBLES + HS;
  static constexpr size_t smem_bytes() { return (size_t)(G::TAB_DOUBLES + WARP_DOUBLES) * 8; }
};

__device__ __forceinline__ void stance_map(int mask, int (&leg_of)[4]) {
  int sf = 0;
#pragma unroll
  for (int leg = 0; leg < 4; ++leg)
    if ((mask >> leg) & 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k == sf) leg_of[k] = leg;
      ++sf;
    }
}

// One warp per QP: gather the stance sub-block of the caller's dense Hessian into shared memory
// (scaled), solve, scatter u.
template <int NS, int N>
__global__ void __launch_bounds__(32 * Geo<NS, N>::TW) dense_solve_kernel(const __grid_constant__ DevParams P, const double* __restrict__ H,
                                                         const double* __restrict__ g, const uint32_t* __restrict__ contact,
                                                         const int* __restrict__ list, const int* __restrict__ count,
                                                         double* __restrict__ u, int32_t* __restrict__ status) {
  using G = Geo<NS, N>;
  using DG = DenseGeo<NS, N>;
  A1MPC_DYN_SMEM(smem);
  const int lane = threadIdx.x & 31;   // one QP per CTA; the CTA is one team of G::TW warps
  Ctx<NS, N> c(smem + G::TAB_DOUBLES, smem, lane);
  double* Hs = smem + G::TAB_DOUBLES + G::WARP_DOUBLES;
  constexpr int n = 12 * N, NV = G::NV, A = G::A;
  const int nq = count[NS];
#pragma unroll 1
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int b = list[q];
    const int mask = contact[b] & 15;
    int leg_of[4] = {0, 0, 0, 0};
    stance_map(mask, leg_of);
    const double* Hb = H + (size_t)b * n * n;
    const double* gb = g + (size_t)b * n;
    // full index of reduced variable v = (step, stance foot, axis)
    auto full = [&](int v) {
      const int s = v / A, r = v - s * A, sf = r / 3, a = r - 3 * sf;
      int leg = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k == sf) leg = leg_of[k];
      return 12 * s + 3 * leg + a;
    };
    double dmax = 0.0;
    bool bad = false;
    for (int v = c.tid; v < NV; v += G::TS) {
      const int fv = full(v);
      const double d = Hb[(size_t)fv * n + fv];
      dmax = fmax(dmax, d);
      bad = bad || !(d > 0.0) || !(fabs(gb[fv]) < 1e300);
    }
    dmax = tmax(c, dmax);
    bad = tany(c, bad);
    if (!bad) {
      const double cs = dmax * FSCALE * FSCALE, hs = FSCALE * FSCALE / cs;
      for (int e = c.tid; e < NV * NV; e += G::TS) {
        const int j = e / NV, i = e - j * NV;
        // symmetrise like OSQP does (osqp-eigen hands over the upper triangle only)
        const int fi = full(i), fj = full(j);
        const double v = (fi <= fj) ? Hb[(size_t)fi * n + fj] : Hb[(size_t)fj * n + fi];
        bad = bad || !(fabs(v) < 1e300);   // every stance entry read: NaN / Inf / huge anywhere -> numerical, zero forces
        Hs[e] = v * hs;
      }
      bad = tany(c, bad);
    }
    int st, iters = 0;
    if (bad) {
      st = A1MPC_STATUS_NUMERICAL;
      for (int i = c.tid; i < G::NPAD; i += G::TS) c.vy[i] = 0.0;
      tsync(c);
    } else {
      const double gsc = FSCALE / (dmax * FSCALE * FSCALE);
      for (int v = c.tid; v < NV; v += G::TS) c.g[v] = gb[full(v)] * gsc;
      tsync(c);
      if (c.wit == 0) fill_padding<NS, N, 0>(c);
      if (G::TW > 1) tsync(c);
      DenseHess<NS, N> hp;
      hp.Hs = Hs;
      st = solve_qp<NS, N, 0, DenseHess<NS, N>, DirectLS<NS, N, DenseHess<NS, N>>>(c, hp, P, iters);
    }
    for (int e = c.tid; e < n; e += G::TS) {
      const int s = e / 12, r = e - 12 * s, leg = r / 3, a = r - 3 * leg;
      double v = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < NS && leg_of[k] == leg && ((mask >> leg) & 1)) v = c.vy[s * A + 3 * k + a] * FSCALE;
      u[(size_t)b * n + e] = v;
    }
    if (c.tid == 0) status[b] = st;
    tsync(c);
  }
}

// compute_grf QP branch on one warp, for one robot: build the 12-variable QP of A1RobotControl.cpp:394-406, solve, rotate.
// The inputs come from four arrays, rot_z / rot row-major and foot leg-major; the 12 forces go to f[(3 * leg + a) * fstride].
// grf_qp_kernel (QP-major caller arrays) and stance_qp_kernel (the record of stance_pack_kernel, batch-major output) both run it.
// EXT (stance_qp_ext_kernel): each stance foot's force is posed in its terrain frame T(n) = [e0 e1 e2] (terrain_col, the frame of the MPC's
// _ext solve, so a foot gets the same pyramid in both modes): column (leg, b) of inertia_inv becomes [e_b ; Rz^T (p_leg x e_b)], the pyramid
// and the 0 <= f_n <= 180 bounds of the unchanged solve act on the local forces, and the output is R^T T u_local.  R I is invariant under
// the orthonormal T.  The normal of leg l is read at nin[(3 l + k) * nld] and normalised as pack_ext_kernel does; a stance foot's normal
// that is not finite or has n_z <= 0 makes the QP NUMERICAL.  Ns: 12 doubles of the warp's shared memory that carry the unit normals
// from the set-up lanes past the solve to the output lanes.
template <int NS, bool EXT = false>
__device__ __forceinline__ int grf_qp_body(const DevParams& P, Ctx<NS, 1>& c, double* Hs, double* Mi, int lane, int mask, const double* acc,
                                           const double* rz, const double* R, const double* ft, double* f, size_t fstride,
                                           const double* nin = nullptr, size_t nld = 0, double* Ns = nullptr) {
  using G = Geo<NS, 1>;
  constexpr int NV = G::NV;
  const double Qd[6] = {1.0, 1.0, 1.0, 400.0, 400.0, 100.0};  // A1RobotControl.cpp:11
  const double Rw = 1e-3;                                      // :12
  int leg_of[4] = {0, 0, 0, 0};
  stance_map(mask, leg_of);
  bool bad = false;
  // inertia_inv (:394-399): rows 0..2 identity blocks, rows 3..5 = Rz^T * skew(foot_i)
  if (lane < 12) {
    const int leg = lane / 3, bb = lane - 3 * leg;
    const double rx = ft[3 * leg], ry = ft[3 * leg + 1], rzz = ft[3 * leg + 2];
    if (EXT) {
      double e[3] = {bb == 0 ? 1.0 : 0.0, bb == 1 ? 1.0 : 0.0, bb == 2 ? 1.0 : 0.0};
      bool nbad = false;
      if ((mask >> leg) & 1) {   // a swing foot's normal is not read
        double n[3] = {nin[(size_t)(3 * leg) * nld], nin[(size_t)(3 * leg + 1) * nld], nin[(size_t)(3 * leg + 2) * nld]};
        const double inv = rsqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        n[0] *= inv; n[1] *= inv; n[2] *= inv;
        if (!(n[2] > 0.0)) { nbad = true; n[0] = 0.0; n[1] = 0.0; n[2] = 1.0; }
        Ns[lane] = bb == 0 ? n[0] : (bb == 1 ? n[1] : n[2]);
        // every column with a constant index, then a select: a lane-dependent index would put n and the frame in local memory
        double e0[3], e1[3], e2[3];
        terrain_col(n, 0, e0); terrain_col(n, 1, e1); terrain_col(n, 2, e2);
#pragma unroll
        for (int a = 0; a < 3; ++a) e[a] = bb == 0 ? e0[a] : (bb == 1 ? e1[a] : e2[a]);
      }
      const double s0 = ry * e[2] - rzz * e[1], s1 = rzz * e[0] - rx * e[2], s2 = rx * e[1] - ry * e[0];   // p x e_b
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        Mi[a * 12 + lane] = e[a];
        Mi[(3 + a) * 12 + lane] = rz[0 * 3 + a] * s0 + rz[1 * 3 + a] * s1 + rz[2 * 3 + a] * s2;  // (Rz^T (p x e_b))[a]
      }
      bad = nbad;
    } else {
      const double s0 = (bb == 0) ? 0.0 : (bb == 1 ? -rzz : ry);
      const double s1 = (bb == 0) ? rzz : (bb == 1 ? 0.0 : -rx);
      const double s2 = (bb == 0) ? -ry : (bb == 1 ? rx : 0.0);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        Mi[a * 12 + lane] = (a == bb) ? 1.0 : 0.0;
        Mi[(3 + a) * 12 + lane] = rz[0 * 3 + a] * s0 + rz[1 * 3 + a] * s1 + rz[2 * 3 + a] * s2;  // (Rz^T S)[a][bb]
      }
    }
    bad = bad || !(fabs(rx) < 1e300) || !(fabs(ry) < 1e300) || !(fabs(rzz) < 1e300);
  }
  if (lane < 6) bad = bad || !(fabs(acc[lane]) < 1e300);
  bad = __any_sync(0xffffffffu, bad);
  __syncwarp();
  auto full = [&](int v) {
    const int sf = v / 3, a = v - 3 * sf;
    int leg = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k == sf) leg = leg_of[k];
    return 3 * leg + a;
  };
  // reduced Hessian / gradient (:400-406): H = R I + M' Q M (no factor 2), g = -M' Q root_acc
  double hv[(NV * NV + 31) / 32];
  double dmax = 0.0;
#pragma unroll
  for (int t = 0; t < (NV * NV + 31) / 32; ++t) {
    const int e = lane + 32 * t;
    hv[t] = 0.0;
    if (e < NV * NV) {
      const int j = e / NV, i = e - j * NV, fi = full(i), fj = full(j);
      double s = (i == j) ? Rw : 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) s = fma(Mi[k * 12 + fi] * Qd[k], Mi[k * 12 + fj], s);
      hv[t] = s;
      if (i == j) dmax = fmax(dmax, s);
    }
  }
  double gv = 0.0;
  if (lane < NV) {
    const int fi = full(lane);
#pragma unroll
    for (int k = 0; k < 6; ++k) gv = fma(Mi[k * 12 + fi] * Qd[k], acc[k], gv);
    gv = -gv;
  }
  dmax = warp_max(dmax);
  __syncwarp();
  int st, iters = 0;
  if (bad) {
    st = A1MPC_STATUS_NUMERICAL;
    for (int i = lane; i < G::NPAD; i += 32) c.vy[i] = 0.0;
    __syncwarp();
  } else {
    const double cs = dmax * FSCALE * FSCALE, hs = FSCALE * FSCALE / cs, gsc = FSCALE / cs;
#pragma unroll
    for (int t = 0; t < (NV * NV + 31) / 32; ++t) {
      const int e = lane + 32 * t;
      if (e < NV * NV) Hs[e] = hv[t] * hs;
    }
    if (lane < NV) c.g[lane] = gv * gsc;
    __syncwarp();
    fill_padding<NS, 1, 0>(c);
    DenseHess<NS, 1> hp;
    hp.Hs = Hs;
    st = solve_qp<NS, 1, 0, DenseHess<NS, 1>, DirectLS<NS, 1, DenseHess<NS, 1>>>(c, hp, P, iters);
  }
  // :439-444  foot_forces_grf = root_rot_mat^T * QPSolution
  if (lane < 4) {
    double fo[3] = {0.0, 0.0, 0.0};
    int sfi = -1;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < NS && leg_of[k] == lane && ((mask >> lane) & 1)) sfi = k;
    if (sfi >= 0) {
      double ux = c.vy[3 * sfi] * FSCALE, uy = c.vy[3 * sfi + 1] * FSCALE, uz = c.vy[3 * sfi + 2] * FSCALE;
      if (EXT) {   // local -> world: T u
        const double n[3] = {Ns[3 * lane], Ns[3 * lane + 1], Ns[3 * lane + 2]};
        double e0[3], e1[3], e2[3];
        terrain_col(n, 0, e0); terrain_col(n, 1, e1); terrain_col(n, 2, e2);
        const double wx = e0[0] * ux + e1[0] * uy + e2[0] * uz, wy = e0[1] * ux + e1[1] * uy + e2[1] * uz, wz = e0[2] * ux + e1[2] * uy + e2[2] * uz;
        ux = wx; uy = wy; uz = wz;
      }
#pragma unroll
      for (int a = 0; a < 3; ++a) fo[a] = R[a] * ux + R[3 + a] * uy + R[6 + a] * uz;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) f[(size_t)(3 * lane + a) * fstride] = fo[a];
  }
  return st;
}

// a1mpc_grf_qp_batch: QP-major caller arrays, the robots of one stance-foot count (classify_kernel's list), one warp each.
template <int NS>
__global__ void __launch_bounds__(32) grf_qp_kernel(const __grid_constant__ DevParams P, const double* __restrict__ root_acc,
                                                    const double* __restrict__ rot_z, const double* __restrict__ rot,
                                                    const double* __restrict__ foot, const uint32_t* __restrict__ contact,
                                                    const int* __restrict__ list, const int* __restrict__ count,
                                                    double* __restrict__ f_body, int32_t* __restrict__ status) {
  using G = Geo<NS, 1>;
  A1MPC_DYN_SMEM(smem);
  const int lane = threadIdx.x;
  Ctx<NS, 1> c(smem + G::TAB_DOUBLES, smem, lane);
  double* Hs = smem + G::TAB_DOUBLES + G::WARP_DOUBLES;
  double* Mi = Hs + DenseGeo<NS, 1>::HS;  // 6 x 12 inertia_inv scratch
  const int nq = count[NS];
#pragma unroll 1
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int b = list[q];
    const int mask = contact[b] & 15;
    const int st = grf_qp_body<NS>(P, c, Hs, Mi, lane, mask, root_acc + (size_t)b * 6, rot_z + (size_t)b * 9, rot + (size_t)b * 9,
                                   foot + (size_t)b * 12, f_body + (size_t)b * 12, 1);
    if (lane == 0) status[b] = st;
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// a1mpc_stance_qp_batch: compute_grf's QP branch from the controller state (A1RobotControl.cpp:321-333, 377-445), batch-major.
// stance_pack_kernel (thread per robot) runs the PD law in front of the QP and writes one STANCE_REC-double record per robot
// (root_acc, rot_z, rot, foot: the arguments of grf_qp_body); stance_qp_kernel<NS> then solves each class like grf_qp_kernel.
// ------------------------------------------------------------------------------------------------
constexpr int STANCE_REC = 36;

struct StanceGains {
  double kd_lin[3], kp_ang[3], kd_ang[3];
  double mass;
};

__global__ void stance_pack_kernel(int B, size_t ld, const double* __restrict__ x0, const double* __restrict__ rot,
                                   const double* __restrict__ rot_z, const double* __restrict__ foot, const uint32_t* __restrict__ contact,
                                   const double* __restrict__ des, const double* __restrict__ kp_linear, const __grid_constant__ StanceGains G,
                                   double* __restrict__ rec, int* __restrict__ list, int* __restrict__ count, double* __restrict__ f_body,
                                   int32_t* __restrict__ status, double* __restrict__ root_acc) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double x[12], d[12], R[9];
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    x[k] = x0[k * ld + b];
    d[k] = des[k * ld + b];
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = rot[k * ld + b];
  // x0: root_euler, root_pos, root_ang_vel, root_lin_vel; des: root_euler_d, root_pos_d, root_lin_vel_d (body), root_ang_vel_d
  double err[3] = {d[0] - x[0], d[1] - x[1], d[2] - x[2]};
  // limit euler error to pi/2 (:327-332, the reference's literals)
  if (err[2] > 3.1415926 * 1.5) err[2] = d[2] - 3.1415926 * 2 - x[2];
  else if (err[2] < -3.1415926 * 1.5) err[2] = d[2] + 3.1415926 * 2 - x[2];
  double acc[6], t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double rtv = R[i] * x[9] + R[3 + i] * x[10] + R[6 + i] * x[11];    // root_rot_mat^T root_lin_vel
    const double rtw = R[i] * x[6] + R[3 + i] * x[7] + R[6 + i] * x[8];      // root_rot_mat^T root_ang_vel
    t[i] = G.kd_lin[i] * (d[6 + i] - rtv);
    acc[3 + i] = G.kp_ang[i] * err[i] + G.kd_ang[i] * (d[9 + i] - rtw);      // :385-389
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)                                                // :380-383
    acc[i] = kp_linear[i * ld + b] * (d[3 + i] - x[3 + i]) + (R[3 * i] * t[0] + R[3 * i + 1] * t[1] + R[3 * i + 2] * t[2]);
  acc[2] += G.mass * 9.8;                                                    // :391
  if (root_acc)
#pragma unroll
    for (int k = 0; k < 6; ++k) root_acc[k * ld + b] = acc[k];
  const int ns = __popc(contact[b] & 15u);
  double* r = rec + (size_t)b * STANCE_REC;
  bool fin = true;
#pragma unroll
  for (int k = 0; k < 6; ++k) { r[k] = acc[k]; fin = fin && fabs(acc[k]) < 1e300; }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const double z = rot_z[k * ld + b];
    r[6 + k] = z; r[15 + k] = R[k];
    fin = fin && fabs(z) < 1e300 && fabs(R[k]) < 1e300;
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    const double p = foot[k * ld + b];
    r[24 + k] = p;
    fin = fin && fabs(p) < 1e300;
  }
  if (ns == 0 || !fin) {   // no stance foot: zero forces by the constraints; non-finite QP data: not posed
#pragma unroll
    for (int k = 0; k < 12; ++k) f_body[k * ld + b] = 0.0;
    status[b] = ns == 0 ? A1MPC_STATUS_NO_CONTACT : A1MPC_STATUS_NUMERICAL;
    return;
  }
  const int slot = atomicAdd(&count[ns], 1);
  list[(size_t)(ns - 1) * B + slot] = b;
}

template <int NS>
__global__ void __launch_bounds__(32) stance_qp_kernel(const __grid_constant__ DevParams P, const double* __restrict__ rec,
                                                       const uint32_t* __restrict__ contact, const int* __restrict__ list,
                                                       const int* __restrict__ count, double* __restrict__ f_body, size_t ld,
                                                       int32_t* __restrict__ status) {
  using G = Geo<NS, 1>;
  A1MPC_DYN_SMEM(smem);
  const int lane = threadIdx.x;
  Ctx<NS, 1> c(smem + G::TAB_DOUBLES, smem, lane);
  double* Hs = smem + G::TAB_DOUBLES + G::WARP_DOUBLES;
  double* Mi = Hs + DenseGeo<NS, 1>::HS;  // 6 x 12 inertia_inv scratch
  const int nq = count[NS];
#pragma unroll 1
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int b = list[q];
    const int mask = contact[b] & 15;
    const double* r = rec + (size_t)b * STANCE_REC;
    const int st = grf_qp_body<NS>(P, c, Hs, Mi, lane, mask, r, r + 6, r + 15, r + 24, f_body + b, ld);
    if (lane == 0) status[b] = st;
    __syncwarp();
  }
}

// a1mpc_stance_qp_batch_ext: stance_qp_kernel with per-foot terrain normals [12][ld] (grf_qp_body<NS, true>); the unit normals are staged
// in 12 doubles behind the inertia_inv scratch
template <int NS>
__global__ void __launch_bounds__(32) stance_qp_ext_kernel(const __grid_constant__ DevParams P, const double* __restrict__ rec,
                                                           const uint32_t* __restrict__ contact, const int* __restrict__ list,
                                                           const int* __restrict__ count, const double* __restrict__ normals,
                                                           double* __restrict__ f_body, size_t ld, int32_t* __restrict__ status) {
  using G = Geo<NS, 1>;
  A1MPC_DYN_SMEM(smem);
  const int lane = threadIdx.x;
  Ctx<NS, 1> c(smem + G::TAB_DOUBLES, smem, lane);
  double* Hs = smem + G::TAB_DOUBLES + G::WARP_DOUBLES;
  double* Mi = Hs + DenseGeo<NS, 1>::HS;  // 6 x 12 inertia_inv scratch
  double* Ns = Mi + 72;                   // 4 x 3 unit normals
  const int nq = count[NS];
#pragma unroll 1
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int b = list[q];
    const int mask = contact[b] & 15;
    const double* r = rec + (size_t)b * STANCE_REC;
    const int st = grf_qp_body<NS, true>(P, c, Hs, Mi, lane, mask, r, r + 6, r + 15, r + 24, f_body + b, ld, normals + b, ld, Ns);
    if (lane == 0) status[b] = st;
    __syncwarp();
  }
}

// the QP constants of compute_grf (A1RobotControl.cpp:13-15); Q and R are literals of grf_qp_body
inline DevParams grf_params() {
  DevParams P;
  memset(&P, 0, sizeof(P));
  P.N = 1; P.max_iter = 40; P.mu = 0.7; P.fzmax = 180.0; P.mu_switch = 1e-9;
  return P;
}

#ifndef A1MPC_EMU
// ------------------------------------------------------------------------------------------------
// host wrappers
// ------------------------------------------------------------------------------------------------
template <int N>
static size_t qp_mats_smem() { return (size_t)(N * 169 + N * 156 + 26) * 8; }

template <int NS, int N>
static cudaError_t dense_attr() {
  return cudaFuncSetAttribute(dense_solve_kernel<NS, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DenseGeo<NS, N>::smem_bytes());
}

cudaError_t dense_setup(int horizon) {
  cudaError_t e;
  if (horizon == 10) {
    if ((e = cudaFuncSetAttribute(qp_mats_kernel<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)qp_mats_smem<10>())) != cudaSuccess) return e;
    if ((e = dense_attr<1, 10>()) != cudaSuccess) return e;
    if ((e = dense_attr<2, 10>()) != cudaSuccess) return e;
    if ((e = dense_attr<3, 10>()) != cudaSuccess) return e;
    if ((e = dense_attr<4, 10>()) != cudaSuccess) return e;
  } else {
    if ((e = cudaFuncSetAttribute(qp_mats_kernel<20>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)qp_mats_smem<20>())) != cudaSuccess) return e;
    if ((e = dense_attr<1, 20>()) != cudaSuccess) return e;
    if ((e = dense_attr<2, 20>()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t dense_qp_mats_launch(const DevParams& P, int B, const double* A_d, const double* B_d_list, const double* x0, const double* x_d,
                                 double* H, double* g, double* A_qp, double* B_qp, cudaStream_t st) {
  if (P.N == 10) qp_mats_kernel<10><<<B, 256, qp_mats_smem<10>(), st>>>(P, B, A_d, B_d_list, x0, x_d, H, g, A_qp, B_qp);
  else qp_mats_kernel<20><<<B, 256, qp_mats_smem<20>(), st>>>(P, B, A_d, B_d_list, x0, x_d, H, g, A_qp, B_qp);
  return cudaGetLastError();
}

template <int NS, int N>
static void dense_launch_one(const DevParams& P, int sm_count, int B, const double* H, const double* g, const uint32_t* contact,
                             const int* list, const int* count, double* u, int32_t* status, cudaStream_t st) {
  int grid = B < sm_count * 4 ? B : sm_count * 4;
  dense_solve_kernel<NS, N><<<grid, 32 * Geo<NS, N>::TW, DenseGeo<NS, N>::smem_bytes(), st>>>(P, H, g, contact, list + (size_t)(NS - 1) * B, count, u, status);
}

cudaError_t dense_solve_launch(const DevParams& P, int sm_count, int B, const double* H, const double* g, const uint32_t* contact, double* u,
                               int32_t* status, int* scratch, cudaStream_t st, int* nlaunch) {
  int* count = scratch;
  int* list = scratch + 8;
  cudaError_t e = cudaMemsetAsync(count, 0, 8 * sizeof(int), st);
  if (e != cudaSuccess) return e;
  const int n = 12 * P.N;
  classify_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, contact, list, count, u, n, status);
  int nl = 1;
  if (P.N == 10) {
    dense_launch_one<4, 10>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    dense_launch_one<3, 10>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    dense_launch_one<2, 10>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    dense_launch_one<1, 10>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    nl += 4;
  } else {
    // 180 x 180 and 240 x 240 dense Hessian + factor exceed shared memory: reported per QP, never approximated
    mark_unsupported_kernel<<<(B + 127) / 128, 128, 0, st>>>(list + (size_t)3 * B, count, 4, u, n, status);
    mark_unsupported_kernel<<<(B + 127) / 128, 128, 0, st>>>(list + (size_t)2 * B, count, 3, u, n, status);
    dense_launch_one<2, 20>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    dense_launch_one<1, 20>(P, sm_count, B, H, g, contact, list, count, u, status, st);
    nl += 4;
  }
  if (nlaunch) *nlaunch = nl;
  return cudaGetLastError();
}

template <int NS>
static cudaError_t grf_launch_one(const DevParams& P, int sm_count, int B, const double* root_acc, const double* rot_z, const double* rot,
                                  const double* foot, const uint32_t* contact, const int* list, const int* count, double* f_body,
                                  int32_t* status, cudaStream_t st) {
  const size_t smem = DenseGeo<NS, 1>::smem_bytes() + 72 * 8;
  cudaError_t e = cudaFuncSetAttribute(grf_qp_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int grid = B < sm_count * 16 ? B : sm_count * 16;
  grf_qp_kernel<NS><<<grid, 32, smem, st>>>(P, root_acc, rot_z, rot, foot, contact, list + (size_t)(NS - 1) * B, count, f_body, status);
  return cudaGetLastError();
}

cudaError_t grf_qp_launch(int sm_count, int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot,
                          const uint32_t* contact, double* f_body, int32_t* status, int* scratch, cudaStream_t st, int* nlaunch) {
  const DevParams P = grf_params();
  int* count = scratch;
  int* list = scratch + 8;
  cudaError_t e = cudaMemsetAsync(count, 0, 8 * sizeof(int), st);
  if (e != cudaSuccess) return e;
  classify_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, contact, list, count, f_body, 12, status);
  if ((e = grf_launch_one<4>(P, sm_count, B, root_acc, rot_z, rot, foot, contact, list, count, f_body, status, st)) != cudaSuccess) return e;
  if ((e = grf_launch_one<3>(P, sm_count, B, root_acc, rot_z, rot, foot, contact, list, count, f_body, status, st)) != cudaSuccess) return e;
  if ((e = grf_launch_one<2>(P, sm_count, B, root_acc, rot_z, rot, foot, contact, list, count, f_body, status, st)) != cudaSuccess) return e;
  if ((e = grf_launch_one<1>(P, sm_count, B, root_acc, rot_z, rot, foot, contact, list, count, f_body, status, st)) != cudaSuccess) return e;
  if (nlaunch) *nlaunch = 5;
  return cudaGetLastError();
}

template <int NS>
static cudaError_t stance_launch_one(const DevParams& P, int sm_count, int B, const double* rec, const uint32_t* contact, const int* list,
                                     const int* count, const double* normals, double* f_body, size_t ld, int32_t* status, cudaStream_t st) {
  int grid = B < sm_count * 16 ? B : sm_count * 16;
  if (normals) {
    const size_t smem = DenseGeo<NS, 1>::smem_bytes() + 84 * 8;
    cudaError_t e = cudaFuncSetAttribute(stance_qp_ext_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    stance_qp_ext_kernel<NS><<<grid, 32, smem, st>>>(P, rec, contact, list + (size_t)(NS - 1) * B, count, normals, f_body, ld, status);
    return cudaGetLastError();
  }
  const size_t smem = DenseGeo<NS, 1>::smem_bytes() + 72 * 8;
  cudaError_t e = cudaFuncSetAttribute(stance_qp_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  stance_qp_kernel<NS><<<grid, 32, smem, st>>>(P, rec, contact, list + (size_t)(NS - 1) * B, count, f_body, ld, status);
  return cudaGetLastError();
}

static size_t stance_lists_bytes(int B) { return ((4 * (size_t)B + 8) * sizeof(int) + 255) & ~(size_t)255; }

size_t stance_scratch_bytes(int B) { return stance_lists_bytes(B) + (size_t)B * STANCE_REC * sizeof(double); }

cudaError_t stance_qp_launch(int sm_count, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                             const uint32_t* contact, const double* des, const double* kp_linear, const double* gains9, double mass,
                             const double* normals, double* f_body, int32_t* status, double* root_acc, void* scratch, cudaStream_t st,
                             int* nlaunch) {
  const DevParams P = grf_params();
  StanceGains G;
  for (int i = 0; i < 3; ++i) { G.kd_lin[i] = gains9[i]; G.kp_ang[i] = gains9[3 + i]; G.kd_ang[i] = gains9[6 + i]; }
  G.mass = mass;
  int* count = static_cast<int*>(scratch);
  int* list = count + 8;
  double* rec = reinterpret_cast<double*>(static_cast<char*>(scratch) + stance_lists_bytes(B));
  cudaError_t e = cudaMemsetAsync(count, 0, 8 * sizeof(int), st);
  if (e != cudaSuccess) return e;
  stance_pack_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, ld, x0, rot, rot_z, foot, contact, des, kp_linear, G, rec, list, count, f_body, status,
                                                       root_acc);
  if ((e = stance_launch_one<4>(P, sm_count, B, rec, contact, list, count, normals, f_body, ld, status, st)) != cudaSuccess) return e;
  if ((e = stance_launch_one<3>(P, sm_count, B, rec, contact, list, count, normals, f_body, ld, status, st)) != cudaSuccess) return e;
  if ((e = stance_launch_one<2>(P, sm_count, B, rec, contact, list, count, normals, f_body, ld, status, st)) != cudaSuccess) return e;
  if ((e = stance_launch_one<1>(P, sm_count, B, rec, contact, list, count, normals, f_body, ld, status, st)) != cudaSuccess) return e;
  if (nlaunch) *nlaunch = 5;
  return cudaGetLastError();
}

#endif  // A1MPC_EMU

}  // namespace a1mpc
