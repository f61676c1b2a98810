// a1mpc_api.cu -- C ABI of the engine (include/a1mpc.h) over the sm_90a kernels.
// No CPU fallback anywhere in this file: every compute entry point launches CUDA kernels or fails.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <algorithm>
#include <initializer_list>

#include "a1mpc_internal.h"
#include "a1mpc_misc.cuh"
#include "a1mpc_estim.cuh"
#include "a1mpc_swing.cuh"
#include "a1mpc_tick.cuh"
#include "a1mpc_gait.cuh"

using namespace a1mpc;

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(A1MPC_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                \
  } while (0)

}  // namespace

extern "C" void a1mpc_internal_nccl_destroy(void* comm);   // a1mpc_nccl.cpp
extern "C" void* a1mpc_internal_gather_begin(a1mpc_handle* h);
extern "C" void a1mpc_internal_gather_end(a1mpc_handle* h);

struct a1mpc_handle {
  int device = 0;
  int sm_count = 0;
  size_t l2_bytes = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t side[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[4] = {nullptr, nullptr, nullptr, nullptr};
  a1mpc_config cfg;
  DevParams P;
  a1mpc::ClassLaunch cls[5];  // index = number of stance feet
  a1mpc::ClassLaunch cls_ext;  // extended path (config 4)
  a1mpc::ClassLaunch cls_sched2;   // its compacted two-feet-per-step class (N = 10; A1MPC_EXT_COMPACT=0 disables it)
  a1mpc::ClassLaunch cls_ext_warm, cls_sched2_warm;   // their warm-started variants (a1mpc_solve_batch_ext_warm, N = 10)
  bool ext_compact = false;
  double* d_rec_ext = nullptr;
  size_t cap_ext = 0;
  // scratch sized for `cap` QPs
  size_t cap = 0;
  double* d_rec = nullptr;
  int* d_count = nullptr;
  // device copies of the batch arrays of a host-pointer call (Stage)
  void* d_side = nullptr;
  size_t side_bytes = 0;
  int* d_lists = nullptr;
  size_t lists_bytes = 0;
  double* d_flush = nullptr;
  size_t flush_elems = 0;
  int64_t launches = 0;
  // optional per-class kernel timing (bench roofline): event pairs on the class streams
  bool prof_on = false;
  int prof_cap = 0, prof_n = 0;
  std::vector<cudaEvent_t> prof_ev;  // [call][class 1..4][begin,end]
  // NCCL (dlopen'ed)
  void* nccl_lib = nullptr;
  void* nccl_comm = nullptr;
  cudaStream_t gather_stream = nullptr;   // the optional final collect runs here, overlapped with the next step's solve
  cudaEvent_t ev_gather_in = nullptr, ev_gather_done = nullptr;
  bool gather_pending = false;
  // fused final collect over peer memory (a1mpc_peer_gather_*)
  struct PeerGather {
    bool connected = false;
    int nranks = 0, rank = 0;
    size_t B = 0;
    void* local = nullptr;                 // this rank's allocation: [nranks][12][B] doubles, then nranks u64 step flags, then an int error word
    double* buf[MAX_PEERS] = {nullptr};    // every rank's gathered buffer as mapped into this process (buf[rank] == local)
    unsigned long long* flags[MAX_PEERS] = {nullptr};
    bool opened[MAX_PEERS] = {false};
    unsigned long long step = 0;
  } peer;
#if A1MPC_TIMELINE
  unsigned long long* tl = nullptr;   // measurement build: timeline records of the class kernels (a1mpc_timeline_attach)
#endif
};

namespace {

int ensure_capacity(a1mpc_handle* h, size_t B) {
  if (B > h->cap) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->d_rec) cudaFree(h->d_rec);
    h->d_rec = nullptr;
    size_t cap = 1024;
    while (cap < B) cap *= 2;
    h->cap = cap;
    CK(cudaMalloc(&h->d_rec, 4 * cap * REC_BYTES));
  }
  return A1MPC_OK;
}

int ensure_side(a1mpc_handle* h, size_t bytes) {
  if (bytes > h->side_bytes) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->d_side) cudaFree(h->d_side);
    h->d_side = nullptr;
    CK(cudaMalloc(&h->d_side, bytes));
    h->side_bytes = bytes;
  }
  return A1MPC_OK;
}

// the extended path's record queues (the general kernel's, then the compacted class's) for h->cap QPs; call after ensure_capacity
int ensure_capacity_ext(a1mpc_handle* h, size_t B) {
  if (B > h->cap_ext) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->d_rec_ext) cudaFree(h->d_rec_ext);
    h->d_rec_ext = nullptr;
    CK(cudaMalloc(&h->d_rec_ext, 2 * h->cap * REC_EXT_BYTES));   // second half: queue of the compacted class
    h->cap_ext = h->cap;
  }
  return A1MPC_OK;
}

int ensure_lists(a1mpc_handle* h, size_t bytes) {
  if (bytes > h->lists_bytes) {
    CK(cudaStreamSynchronize(h->stream));
    if (h->d_lists) cudaFree(h->d_lists);
    h->d_lists = nullptr;
    CK(cudaMalloc(&h->d_lists, bytes));
    h->lists_bytes = bytes;
  }
  return A1MPC_OK;
}

bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The one path by which the batch arrays of an entry point reach its kernels.  The call declares each array (in, out or in/out:
// rows x B elements of 4 or 8 bytes, leading dimension ld in the caller's memory), then begin() classifies every non-NULL array
// once: they must all be host or all device memory, because a host pointer dereferenced by a kernel is a sticky fault for the
// whole CUDA context.  A mix is rejected before anything is enqueued, and so is a device pointer among the batch-uniform
// parameters that the call reads on the host.  Device arrays go to the kernel as they are and the call stays asynchronous.
// Host arrays get one dense [rows][B] slot each in h->d_side: begin() copies the inputs in and points the call's variable at the
// slot, finish() copies the outputs back and synchronises the stream once.
class Stage {
 public:
  Stage(a1mpc_handle* h, int B) : h_(h), B_((size_t)B) { arrays_.reserve(16); }   // update_plan declares the most: 15
  template <class T> void in(T*& p, size_t rows, size_t esz = sizeof(T)) { add(p, IN, rows, esz, B_); }
  template <class T> void in(T*& p, size_t rows, size_t esz, size_t ld) { add(p, IN, rows, esz, ld); }
  template <class T> void out(T*& p, size_t rows, size_t esz = sizeof(T)) { add(p, OUT, rows, esz, B_); }
  template <class T> void out(T*& p, size_t rows, size_t esz, size_t ld) { add(p, OUT, rows, esz, ld); }
  template <class T> void inout(T*& p, size_t rows, size_t esz = sizeof(T)) { add(p, INOUT, rows, esz, B_); }
  template <class T> void inout(T*& p, size_t rows, size_t esz, size_t ld) { add(p, INOUT, rows, esz, ld); }
  // a batch array this call does not read: its side is checked, nothing is copied
  void unused(const void* p) { arrays_.push_back({nullptr, nullptr, const_cast<void*>(p), 0, 0, 0, UNUSED, nullptr}); }
  // a batch-uniform parameter read by the call itself on the host
  void host_param(const void* p, const char* name) { params_.push_back({p, name}); }
  bool host() const { return host_; }

  int begin() {
    bool first = true;
    for (const Array& a : arrays_) {
      if (!a.user) continue;
      const bool host = !is_device_ptr(a.user);
      if (first) {
        host_ = host;
        first = false;
      } else if (host != host_) {
        return fail(A1MPC_EINVAL, "batch arrays must be all-host or all-device");
      }
    }
    for (const Param& p : params_)
      if (is_device_ptr(p.ptr)) return fail(A1MPC_EINVAL, std::string(p.name) + " must be a host array (batch-uniform parameter)");
    if (!host_) return A1MPC_OK;
    size_t bytes = 0;
    for (const Array& a : arrays_)
      if (a.user && a.dir != UNUSED) bytes += pad(a.rows * B_ * a.esz);
    int rc;
    if ((rc = ensure_side(h_, bytes))) return rc;
    char* cur = static_cast<char*>(h_->d_side);
    for (Array& a : arrays_) {
      if (!a.user || a.dir == UNUSED) continue;
      a.slot = cur;
      cur += pad(a.rows * B_ * a.esz);
      a.point(a.var, a.slot);
      if (a.dir != OUT && (rc = copy(a, cudaMemcpyHostToDevice))) return rc;
    }
    return A1MPC_OK;
  }

  int finish() {
    if (!host_) return A1MPC_OK;
    int rc;
    for (const Array& a : arrays_)
      if (a.user && (a.dir == OUT || a.dir == INOUT) && (rc = copy(a, cudaMemcpyDeviceToHost))) return rc;
    CK(cudaStreamSynchronize(h_->stream));
    return A1MPC_OK;
  }

 private:
  enum Dir { IN, OUT, INOUT, UNUSED };
  struct Array {
    void* var;                     // the call's pointer variable, pointed at the slot in host mode
    void (*point)(void*, char*);
    void* user;                    // the caller's array
    size_t rows, esz, ld;
    Dir dir;
    char* slot;
  };
  struct Param { const void* ptr; const char* name; };
  static size_t pad(size_t b) { return (b + 255) & ~(size_t)255; }

  template <class T>
  void add(T*& p, Dir dir, size_t rows, size_t esz, size_t ld) {
    arrays_.push_back({&p, [](void* var, char* slot) { *static_cast<T**>(var) = reinterpret_cast<T*>(slot); },
                       const_cast<void*>(static_cast<const void*>(p)), rows, esz, ld, dir, nullptr});
  }

  int copy(const Array& a, cudaMemcpyKind kind) {
    const bool h2d = kind == cudaMemcpyHostToDevice;
    void* dst = h2d ? a.slot : a.user;
    const void* src = h2d ? a.user : a.slot;
    const size_t row = B_ * a.esz, user_pitch = a.ld * a.esz;
    if (a.ld == B_) CK(cudaMemcpyAsync(dst, src, a.rows * row, kind, h_->stream));
    else CK(cudaMemcpy2DAsync(dst, h2d ? row : user_pitch, src, h2d ? user_pitch : row, row, a.rows, kind, h_->stream));
    return A1MPC_OK;
  }

  a1mpc_handle* h_;
  size_t B_;
  bool host_ = false;
  std::vector<Array> arrays_;
  std::vector<Param> params_;
};

// enqueue the fused path on device-resident SoA data
void attach_peers(a1mpc_handle* h, int B, DevOutputs& d) {
  d.npeer = 0; d.rank = 0; d.peer_ld = 0;
  for (int p = 0; p < MAX_PEERS; ++p) d.peer[p] = nullptr;
  if (h->peer.connected && (size_t)B == h->peer.B) {
    d.npeer = h->peer.nranks; d.rank = h->peer.rank; d.peer_ld = h->peer.B;
    for (int p = 0; p < h->peer.nranks; ++p) d.peer[p] = h->peer.buf[p];
  }
}

int peer_signal(a1mpc_handle* h, int B) {
  if (!(h->peer.connected && (size_t)B == h->peer.B)) return A1MPC_OK;
  PeerFlags pf;
  for (int p = 0; p < MAX_PEERS; ++p) pf.p[p] = h->peer.flags[p];
  h->peer.step++;
  peer_signal_kernel<<<1, 32, 0, h->stream>>>(pf, h->peer.nranks, h->peer.rank, h->peer.step);
  h->launches++;
  CK(cudaGetLastError());
  return A1MPC_OK;
}

// runs: the multi-rate tick's run counters (a1mpc_tick_set_mpc_period), whose robots that are not due this run the pack kernel skips;
// such a solve does not take part in the fused collect
int enqueue_solve(a1mpc_handle* h, int B, const DevInputs& din, const DevOutputs& dout_in, uint32_t* warm = nullptr, int shift = 0,
                  const uint32_t* runs = nullptr, int period = 1) {
  DevOutputs dout = dout_in;
  attach_peers(h, runs ? -1 : B, dout);
#if A1MPC_TIMELINE
  dout.tl = h->tl;
#endif
  CK(cudaMemsetAsync(h->d_count, 0, 16 * sizeof(int), h->stream));
  if (runs) pack_due_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(din, B, h->d_rec, (int)h->cap, h->d_count, dout, h->cfg.horizon, runs, period);
  else pack_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(din, B, h->d_rec, (int)h->cap, h->d_count, dout, h->cfg.horizon);
  h->launches++;
  CK(cudaEventRecord(h->ev_fork, h->stream));
  const int N = h->cfg.horizon;
  // heaviest class first, each class on its own stream so that the few long 4-stance solves overlap
  // the many short trot solves
  for (int ns = 4; ns >= 1; --ns) {
    cudaStream_t st = h->side[ns - 1];
    CK(cudaStreamWaitEvent(st, h->ev_fork, 0));
    const double* rec = h->d_rec + (size_t)(ns - 1) * h->cap * REC_DOUBLES;
    const bool prof = h->prof_on && h->prof_n < h->prof_cap;
    if (prof) CK(cudaEventRecord(h->prof_ev[((size_t)h->prof_n * 4 + (ns - 1)) * 2 + 0], st));
    if (!h->cls[ns].supported) unsupported_kernel<<<(B + 127) / 128, 128, 0, st>>>(rec, h->d_count, ns, dout, N);
    else if (N == 10 && warm) fused_launch_n10_warm(ns, h->cls[ns], st, B, h->P, rec, h->d_count, dout, warm, shift);
    else if (N == 10) fused_launch_n10(ns, h->cls[ns], st, B, h->P, rec, h->d_count, dout);
    else fused_launch_n20(ns, h->cls[ns], st, B, h->P, rec, h->d_count, dout);
    h->launches++;
    if (prof) CK(cudaEventRecord(h->prof_ev[((size_t)h->prof_n * 4 + (ns - 1)) * 2 + 1], st));
    CK(cudaEventRecord(h->ev_join[ns - 1], st));
    CK(cudaStreamWaitEvent(h->stream, h->ev_join[ns - 1], 0));
  }
  if (h->prof_on && h->prof_n < h->prof_cap) h->prof_n++;
  CK(cudaGetLastError());
  if (runs) return A1MPC_OK;
  return peer_signal(h, B);   // fused collect: publish this call's step number to every rank (no-op when not connected)
}

// the same on a schedule (dsched) and / or terrain normals (dnorm): a1mpc_solve_batch_ext and _ext_warm
int enqueue_solve_ext(a1mpc_handle* h, int B, const DevInputs& di, const uint32_t* dsched, const double* dnorm, const DevOutputs& dout_in,
                      uint32_t* warm, int shift, const uint32_t* runs = nullptr, int period = 1) {
  const int N = h->cfg.horizon;
  int rc;
  if ((rc = ensure_capacity_ext(h, B))) return rc;
  DevOutputs dout = dout_in;
  attach_peers(h, -1, dout);   // the fused collect is wired to a1mpc_solve_batch / _warm only
#if A1MPC_TIMELINE
  dout.tl = h->tl;
#endif
  CK(cudaMemsetAsync(h->d_count, 0, 16 * sizeof(int), h->stream));
  if (warm) {   // robots without any contact are answered by the pack kernel and store no guess
    if (runs) warm_forget_no_contact_due_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, B, warm, N, runs, period);
    else warm_forget_no_contact_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, B, warm, N);
    h->launches++;
  }
  if (h->ext_compact && dsched) {
    if (runs)
      pack_ext2_due_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, dnorm, B, h->d_rec_ext, (int)h->cap_ext, h->d_count, dout, N, runs, period);
    else
      pack_ext2_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, dnorm, B, h->d_rec_ext, (int)h->cap_ext, h->d_count, dout, N);
    const double* rec2 = h->d_rec_ext + h->cap_ext * REC_EXT_DOUBLES;
    if (warm) {
      ext_warm_launch(h->cls_ext_warm, h->stream, B, h->P, h->d_rec_ext, h->d_count, dout, warm, shift);
      sched2_warm_launch(h->cls_sched2_warm, h->stream, B, h->P, rec2, h->d_count, dout, warm, shift);
    } else {
      ext_launch(N, h->cls_ext, h->stream, B, h->P, h->d_rec_ext, h->d_count, dout);
      sched2_launch(h->cls_sched2, h->stream, B, h->P, rec2, h->d_count, dout);
    }
    h->launches += 3;
  } else {
    if (runs) pack_ext_due_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, dnorm, B, h->d_rec_ext, h->d_count, dout, N, runs, period);
    else pack_ext_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(di, dsched, dnorm, B, h->d_rec_ext, h->d_count, dout, N);
    if (warm) ext_warm_launch(h->cls_ext_warm, h->stream, B, h->P, h->d_rec_ext, h->d_count, dout, warm, shift);
    else ext_launch(N, h->cls_ext, h->stream, B, h->P, h->d_rec_ext, h->d_count, dout);
    h->launches += 2;
  }
  CK(cudaGetLastError());
  return A1MPC_OK;
}

// a1mpc_solve_batch, _warm, _ext and _ext_warm.  ext: schedule and / or normals (NULL, or both fields NULL: the plain solve);
// warm_start: the _warm calls, with the caller's `warm` buffer and `shift`
int solve_impl(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_inputs_ext* ext, const a1mpc_outputs* out, bool warm_start,
               void* warm, int shift) {
  if (!h || !in || !out || (warm_start && !warm)) return fail(A1MPC_EINVAL, "null argument");
  if (ext && !ext->contact_sched && !ext->normals) ext = nullptr;
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!in->x0 || !in->rot || !in->foot || !in->ref || !in->contact || !out->f_body || !out->status) return fail(A1MPC_EINVAL, "null input/output array");
  if (in->ld < (size_t)B || out->ld < (size_t)B) return fail(A1MPC_EINVAL, "ld < B");
  const int N = h->cfg.horizon;
  if (warm_start && N != 10) return fail(A1MPC_EINVAL, "warm start is implemented for horizon 10 (see include/a1mpc.h)");
  if (warm_start && (shift < 0 || shift > N)) return fail(A1MPC_EINVAL, "shift out of range");
  if (ext && ext->normals)
    for (int i = 0; i < 4; ++i)
      if (h->cfg.r[3 * i] != h->cfg.r[3 * i + 1] || h->cfg.r[3 * i] != h->cfg.r[3 * i + 2])
        return fail(A1MPC_EINVAL, "terrain normals need isotropic r weights per foot (r[3i] == r[3i+1] == r[3i+2])");
  CK(cudaSetDevice(h->device));
  if (warm_start && !is_device_ptr(warm)) return fail(A1MPC_EINVAL, "warm must be device memory (a1mpc_device_alloc)");
  const int f32 = (h->cfg.precision == 32) ? 1 : 0;   // fp32 arrays at the boundary, fp64 inside
  const size_t es = f32 ? 4 : 8;
  DevInputs di{in->x0, in->rot, in->foot, in->ref, in->contact, in->ld, f32};
  DevOutputs dout{out->f_body, out->status, out->iters, out->u_full, out->ld, f32};
  const uint32_t* dsched = ext ? ext->contact_sched : nullptr;
  const double* dnorm = ext ? ext->normals : nullptr;
  Stage st(h, B);
  st.in(di.x0, 12, es, in->ld); st.in(di.rot, 9, es, in->ld); st.in(di.foot, 12, es, in->ld); st.in(di.ref, 9, es, in->ld);
  st.in(di.contact, 1);
  st.in(dsched, N, 4, in->ld); st.in(dnorm, 12, es, in->ld);
  st.out(dout.f_body, 12, es, out->ld); st.out(dout.status, 1); st.out(dout.iters, 1); st.out(dout.u_full, 12 * N, es, out->ld);
  int rc;
  if ((rc = st.begin())) return rc;
  if (st.host()) di.ld = dout.ld = (size_t)B;
  if ((rc = ensure_capacity(h, B))) return rc;
  uint32_t* w = static_cast<uint32_t*>(warm);
  rc = ext ? enqueue_solve_ext(h, B, di, dsched, dnorm, dout, w, shift) : enqueue_solve(h, B, di, dout, w, shift);
  if (rc) return rc;
  return st.finish();
}

int enqueue_ekf_update(a1mpc_handle* h, int B, double* state, EkfParams P, const uint32_t* movement_mode, const double* imu_acc,
                       const double* imu_ang_vel, const double* rot, const double* foot_pos_rel, const double* foot_vel_rel, const double* foot_force,
                       double* root_pos, double* root_lin_vel, uint32_t* estimated_contacts, int32_t* status) {
  static bool attr_set[64] = {};
  const size_t smem = (size_t)EKF_WPC * EKF_WARP_DOUBLES * sizeof(double);
  if (h->device < 64 && !attr_set[h->device]) {
    CK(cudaFuncSetAttribute(ekf_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[h->device] = true;
  }
  int grid = (B + EKF_WPC - 1) / EKF_WPC;
  if (grid > h->sm_count * 2) grid = h->sm_count * 2;
  ekf_update_kernel<<<grid, 32 * EKF_WPC, smem, h->stream>>>(B, P, state, movement_mode, imu_acc, imu_ang_vel, rot, foot_pos_rel, foot_vel_rel,
                                                             foot_force, root_pos, root_lin_vel, estimated_contacts, status);
  h->launches++;
  CK(cudaGetLastError());
  return A1MPC_OK;
}

}  // namespace

extern "C" {

const char* a1mpc_last_error(void) { return g_err.c_str(); }

int a1mpc_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

void a1mpc_default_config(a1mpc_config* c) {
  std::memset(c, 0, sizeof(*c));
  c->horizon = 10;
  c->precision = 64;
  c->dt = 0.0025;
  c->mu = 0.3;
  c->fz_min = 0.0;
  c->fz_max = 180.0;
  c->mass = 12.0;
  c->inertia[0] = 0.0158533; c->inertia[4] = 0.0377999; c->inertia[8] = 0.0456542;
  const double q[13] = {20, 10, 1, 0, 0, 420, 0.05, 0.05, 0.05, 30, 30, 10, 0};
  for (int i = 0; i < 13; ++i) c->q[i] = q[i];
  for (int i = 0; i < 12; ++i) c->r[i] = 1e-7;
  c->max_iter = 0;
  c->tol = 0.0;
}

int a1mpc_create(a1mpc_handle** out, const a1mpc_config* cfg, int device) {
  if (!out || !cfg) return fail(A1MPC_EINVAL, "null argument");
  *out = nullptr;
  if (cfg->horizon != 10 && cfg->horizon != 20) return fail(A1MPC_EINVAL, "horizon must be 10 or 20");
  if (cfg->precision != 64 && cfg->precision != 32) return fail(A1MPC_EINVAL, "precision must be 64 or 32 (see include/a1mpc.h)");
  if (!(cfg->fz_min == 0.0)) return fail(A1MPC_EINVAL, "fz_min must be 0 (the reference hard-codes it, ConvexMpc.cpp:223)");
  if (!(cfg->mu > 0.0) || !(cfg->fz_max > 0.0) || !(cfg->mass > 0.0) || !(cfg->dt > 0.0)) return fail(A1MPC_EINVAL, "mu, fz_max, mass, dt must be positive");
  for (int i = 0; i < 12; ++i)
    if (!(cfg->r[i] > 0.0)) return fail(A1MPC_EINVAL, "r weights must be positive (H must be positive definite)");
  for (int i = 0; i < 13; ++i)
    if (!(cfg->q[i] >= 0.0)) return fail(A1MPC_EINVAL, "q weights must be non-negative");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    return fail(A1MPC_ENODEVICE, "no CUDA device available (this engine has no CPU fallback)");
  }
  if (device < 0 || device >= ndev) return fail(A1MPC_EINVAL, "device index out of range");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  // architecture-specific sm_90a code loads on compute capability 9.0 and nothing else
  if (prop.major != 9 || prop.minor != 0) return fail(A1MPC_ENODEVICE, std::string("device is sm_") + std::to_string(prop.major * 10 + prop.minor) + "; this library is built for sm_90a (H100) only");
  a1mpc_handle* h = new a1mpc_handle();
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  h->l2_bytes = (size_t)prop.l2CacheSize;
  h->cfg = *cfg;
  DevParams& P = h->P;
  P.N = cfg->horizon;
  P.max_iter = cfg->max_iter > 0 ? cfg->max_iter : 40;
  P.dt = cfg->dt; P.mu = cfg->mu; P.fzmax = cfg->fz_max; P.mass = cfg->mass;
  P.mu_switch = cfg->tol > 0.0 ? cfg->tol : MU_SWITCH_DEFAULT;
  for (int i = 0; i < 9; ++i) P.inertia[i] = cfg->inertia[i];
  for (int i = 0; i < 13; ++i) P.q2[i] = 2.0 * cfg->q[i];
  for (int i = 0; i < 12; ++i) P.r2[i] = 2.0 * cfg->r[i];
  int rc = A1MPC_OK;
  auto bail = [&](int code) { a1mpc_destroy(h); return code; };
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(A1MPC_ECUDA, "stream create failed"));
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  for (int i = 0; i < 4; ++i) {
    // the classes with more stance feet take longer per QP: their CTAs are placed first
    const int prio = (i >= 2) ? prio_hi : prio_lo;
    if (cudaStreamCreateWithPriority(&h->side[i], cudaStreamNonBlocking, prio) != cudaSuccess) return bail(fail(A1MPC_ECUDA, "stream create failed"));
    if (cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming) != cudaSuccess) return bail(fail(A1MPC_ECUDA, "event create failed"));
  }
  if (cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess) return bail(fail(A1MPC_ECUDA, "event create failed"));
  if (cudaMalloc(&h->d_count, 16 * sizeof(int)) != cudaSuccess) return bail(fail(A1MPC_ENOMEM, "cudaMalloc failed"));
  {
    cudaError_t e = (cfg->horizon == 10) ? fused_setup_n10(h->sm_count, h->cls) : fused_setup_n20(h->sm_count, h->cls);
    if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("kernel setup: ") + cudaGetErrorString(e)));
    e = ext_setup(cfg->horizon, h->sm_count, h->cls_ext);
    if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("ext kernel setup: ") + cudaGetErrorString(e)));
    if (cfg->horizon == 10) {
      e = ext_warm_setup(h->sm_count, h->cls_ext_warm);
      if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("warm ext kernel setup: ") + cudaGetErrorString(e)));
    }
    {   // schedules with two stance feet in every step run on the compact direct kernel (a1mpc_sched.cuh): a problem the size of
        // the trot problem instead of the general 4-foot one.  A1MPC_EXT_COMPACT=0 keeps everything on the general kernel (A/B).
      const char* ev = std::getenv("A1MPC_EXT_COMPACT");
      if (!(ev && ev[0] == '0') && cfg->horizon == 10) {
        e = sched2_setup(h->sm_count, h->cls_sched2);
        if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("compact ext kernel setup: ") + cudaGetErrorString(e)));
        e = sched2_warm_setup(h->sm_count, h->cls_sched2_warm);
        if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("warm compact ext kernel setup: ") + cudaGetErrorString(e)));
        h->ext_compact = true;
      }
    }
    e = dense_setup(cfg->horizon);
    if (e != cudaSuccess) return bail(fail(A1MPC_ECUDA, std::string("dense kernel setup: ") + cudaGetErrorString(e)));
  }
  (void)rc;
  *out = h;
  return A1MPC_OK;
}

int a1mpc_destroy(a1mpc_handle* h) {
  if (!h) return A1MPC_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->gather_stream) cudaStreamSynchronize(h->gather_stream);
  if (h->nccl_comm) { a1mpc_internal_nccl_destroy(h->nccl_comm); h->nccl_comm = nullptr; }   // before its streams go away
  a1mpc_peer_gather_destroy(h);
  auto fr = [](void* p) { if (p) cudaFree(p); };
  fr(h->d_rec); fr(h->d_count); fr(h->d_side); fr(h->d_flush); fr(h->d_lists); fr(h->d_rec_ext);
  for (int i = 0; i < 4; ++i) {
    if (h->side[i]) cudaStreamDestroy(h->side[i]);
    if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
  }
  for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
  if (h->gather_stream) { cudaStreamSynchronize(h->gather_stream); cudaStreamDestroy(h->gather_stream); cudaEventDestroy(h->ev_gather_in); cudaEventDestroy(h->ev_gather_done); }
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return A1MPC_OK;
}

int a1mpc_solve_batch(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_outputs* out) {
  return solve_impl(h, B, in, nullptr, out, false, nullptr, 0);
}

size_t a1mpc_warm_bytes(const a1mpc_handle* h, int B) {
  if (!h || B <= 0) return 0;
  return (size_t)B * (size_t)(WARM_HDR + 4 * h->cfg.horizon) * sizeof(uint32_t);
}

int a1mpc_warm_reset(a1mpc_handle* h, void* warm, int B) {
  if (!h || !warm || B <= 0) return fail(A1MPC_EINVAL, "null argument");
  if (!is_device_ptr(warm)) return fail(A1MPC_EINVAL, "warm must be device memory (a1mpc_device_alloc)");
  CK(cudaSetDevice(h->device));
  CK(cudaMemsetAsync(warm, 0, a1mpc_warm_bytes(h, B), h->stream));
  return A1MPC_OK;
}

int a1mpc_solve_batch_warm(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_outputs* out, void* warm, int shift) {
  return solve_impl(h, B, in, nullptr, out, true, warm, shift);
}

int a1mpc_solve_batch_ext(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_inputs_ext* ext, const a1mpc_outputs* out) {
  return solve_impl(h, B, in, ext, out, false, nullptr, 0);
}

int a1mpc_solve_batch_ext_warm(a1mpc_handle* h, int B, const a1mpc_inputs* in, const a1mpc_inputs_ext* ext, const a1mpc_outputs* out, void* warm,
                               int shift) {
  return solve_impl(h, B, in, ext, out, true, warm, shift);
}

int a1mpc_build_qp_batch(a1mpc_handle* h, int B, const a1mpc_inputs* in, double* H, double* g, double* lb, double* ub) {
  if (!h || !in) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!in->x0 || !in->rot || !in->foot || !in->ref || !in->contact) return fail(A1MPC_EINVAL, "null input array");
  if ((lb == nullptr) != (ub == nullptr)) return fail(A1MPC_EINVAL, "lb and ub must be given together");
  CK(cudaSetDevice(h->device));
  const int N = h->cfg.horizon, n = 12 * N, m = 20 * N;
  DevInputs di{in->x0, in->rot, in->foot, in->ref, in->contact, in->ld};
  Stage st(h, B);
  st.in(di.x0, 12, 8, in->ld); st.in(di.rot, 9, 8, in->ld); st.in(di.foot, 12, 8, in->ld); st.in(di.ref, 9, 8, in->ld);
  st.in(di.contact, 1);
  st.out(H, (size_t)n * n); st.out(g, n); st.out(lb, m); st.out(ub, m);
  int rc;
  if ((rc = st.begin())) return rc;
  if (st.host()) di.ld = (size_t)B;
  {
    cudaError_t e = build_dense_launch(h->P, di, B, H, g, lb, ub, h->stream);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("build kernel: ") + cudaGetErrorString(e));
    h->launches++;
  }
  return st.finish();
}

static int qp_mats_impl(a1mpc_handle* h, int B, const double* A_d, const double* B_d_list, const double* x0, const double* x_d,
                        double* H, double* g, double* A_qp, double* B_qp) {
  if (!h || !A_d || !B_d_list || !x0 || !x_d || (!H && !g && !A_qp && !B_qp)) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  const int N = h->cfg.horizon, n = 12 * N;
  Stage st(h, B);
  st.in(A_d, 169); st.in(B_d_list, 13 * N * 12); st.in(x0, 13); st.in(x_d, 13 * N);
  st.out(H, (size_t)n * n); st.out(g, n); st.out(A_qp, 13 * N * 13); st.out(B_qp, 13 * N * n);
  int rc;
  if ((rc = st.begin())) return rc;
  {
    cudaError_t e = dense_qp_mats_launch(h->P, B, A_d, B_d_list, x0, x_d, H, g, A_qp, B_qp, h->stream);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("qp_mats kernel: ") + cudaGetErrorString(e));
    h->launches += 1;
  }
  return st.finish();
}

int a1mpc_qp_mats_batch(a1mpc_handle* h, int B, const double* A_d, const double* B_d_list, const double* x0, const double* x_d,
                        double* H, double* g) {
  if (!H && !g) return fail(A1MPC_EINVAL, "null argument");
  return qp_mats_impl(h, B, A_d, B_d_list, x0, x_d, H, g, nullptr, nullptr);
}

int a1mpc_qp_rollout_batch(a1mpc_handle* h, int B, const double* A_d, const double* B_d_list, const double* x0, const double* x_d,
                           double* A_qp, double* B_qp, double* H, double* g) {
  return qp_mats_impl(h, B, A_d, B_d_list, x0, x_d, H, g, A_qp, B_qp);
}

int a1mpc_solve_dense_batch(a1mpc_handle* h, int B, const double* H, const double* g, const uint32_t* contact, double* u, int32_t* status) {
  if (!h || !H || !g || !contact || !u || !status) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  const int N = h->cfg.horizon, n = 12 * N;
  Stage st(h, B);
  st.in(H, (size_t)n * n); st.in(g, n); st.in(contact, 1);
  st.out(u, n); st.out(status, 1);
  int rc;
  if ((rc = st.begin())) return rc;
  if ((rc = ensure_lists(h, (4 * (size_t)B + 8) * sizeof(int)))) return rc;
  {
    int nl = 0;
    cudaError_t e = dense_solve_launch(h->P, h->sm_count, B, H, g, contact, u, status, h->d_lists, h->stream, &nl);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("dense solve kernels: ") + cudaGetErrorString(e));
    h->launches += nl;
  }
  return st.finish();
}

int a1mpc_grf_qp_batch(a1mpc_handle* h, int B, const double* root_acc, const double* rot_z, const double* rot, const double* foot,
                       const uint32_t* contact, double* f_body, int32_t* status) {
  if (!h || !root_acc || !rot_z || !rot || !foot || !contact || !f_body || !status) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(root_acc, 6); st.in(rot_z, 9); st.in(rot, 9); st.in(foot, 12); st.in(contact, 1);
  st.out(f_body, 12); st.out(status, 1);
  int rc;
  if ((rc = st.begin())) return rc;
  if ((rc = ensure_lists(h, (4 * (size_t)B + 8) * sizeof(int)))) return rc;
  {
    int nl = 0;
    cudaError_t e = grf_qp_launch(h->sm_count, B, root_acc, rot_z, rot, foot, contact, f_body, status, h->d_lists, h->stream, &nl);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("grf_qp kernels: ") + cudaGetErrorString(e));
    h->launches += nl;
  }
  return st.finish();
}

}  // extern "C"

// a1mpc_stance_qp_batch, and with normals (not NULL) a1mpc_stance_qp_batch_ext
static int stance_qp_impl(a1mpc_handle* h, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                          const uint32_t* contact, const double* des, const double* kp_linear, const double* kd_linear, const double* kp_angular,
                          const double* kd_angular, const double* normals, double* f_body, int32_t* status, double* root_acc) {
  if (!h || !x0 || !rot || !rot_z || !foot || !contact || !des || !kp_linear || !kd_linear || !kp_angular || !kd_angular || !f_body || !status)
    return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (ld < (size_t)B) return fail(A1MPC_EINVAL, "ld < B");
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(x0, 12, 8, ld); st.in(rot, 9, 8, ld); st.in(rot_z, 9, 8, ld); st.in(foot, 12, 8, ld); st.in(contact, 1);
  st.in(des, 12, 8, ld); st.in(kp_linear, 3, 8, ld); st.in(normals, 12, 8, ld);
  st.out(f_body, 12, 8, ld); st.out(status, 1); st.out(root_acc, 6, 8, ld);
  st.host_param(kd_linear, "kd_linear"); st.host_param(kp_angular, "kp_angular"); st.host_param(kd_angular, "kd_angular");
  int rc;
  if ((rc = st.begin())) return rc;
  const size_t kld = st.host() ? (size_t)B : ld;
  if ((rc = ensure_lists(h, stance_scratch_bytes(B)))) return rc;
  double gains[9];
  for (int i = 0; i < 3; ++i) { gains[i] = kd_linear[i]; gains[3 + i] = kp_angular[i]; gains[6 + i] = kd_angular[i]; }
  {
    int nl = 0;
    cudaError_t e = stance_qp_launch(h->sm_count, B, kld, x0, rot, rot_z, foot, contact, des, kp_linear, gains, h->cfg.mass, normals, f_body,
                                     status, root_acc, h->d_lists, h->stream, &nl);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("stance_qp kernels: ") + cudaGetErrorString(e));
    h->launches += nl;
  }
  return st.finish();
}

extern "C" {

int a1mpc_stance_qp_batch(a1mpc_handle* h, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                          const uint32_t* contact, const double* des, const double* kp_linear, const double* kd_linear, const double* kp_angular,
                          const double* kd_angular, double* f_body, int32_t* status, double* root_acc) {
  return stance_qp_impl(h, B, ld, x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, nullptr, f_body, status,
                        root_acc);
}

int a1mpc_stance_qp_batch_ext(a1mpc_handle* h, int B, size_t ld, const double* x0, const double* rot, const double* rot_z, const double* foot,
                              const uint32_t* contact, const double* des, const double* kp_linear, const double* kd_linear,
                              const double* kp_angular, const double* kd_angular, const double* normals, double* f_body, int32_t* status,
                              double* root_acc) {
  return stance_qp_impl(h, B, ld, x0, rot, rot_z, foot, contact, des, kp_linear, kd_linear, kp_angular, kd_angular, normals, f_body, status,
                        root_acc);
}

int a1mpc_joint_torques_batch(a1mpc_handle* h, int B, const double* f_grf, const double* f_kin, const double* jac, const uint32_t* contact,
                              const double* km_foot, const double* torques_gravity, double* tau) {
  if (!h || !f_grf || !f_kin || !jac || !contact || !km_foot || !torques_gravity || !tau) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(f_grf, 12); st.in(f_kin, 12); st.in(jac, 36); st.in(contact, 1);
  st.inout(tau, 12);
  st.host_param(km_foot, "km_foot"); st.host_param(torques_gravity, "torques_gravity");
  int rc;
  if ((rc = st.begin())) return rc;
  TorqueParams P;
  for (int i = 0; i < 3; ++i) P.km[i] = km_foot[i];
  for (int i = 0; i < 12; ++i) P.tg[i] = torques_gravity[i];
  joint_torques_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, f_grf, f_kin, jac, contact, P, tau);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_update_plan_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, double* gait_counter, const double* gait_counter_speed,
                            const uint32_t* movement_mode, const double* lin_vel, const double* lin_vel_d, const double* rot_z,
                            const double* rot, const double* root_pos, uint32_t* plan_contacts, uint32_t* contact_sched,
                            double* t_rel, double* t_abs, double* t_world) {
  if (!h || !gp || !gait_counter || !gait_counter_speed || !movement_mode || !plan_contacts) return fail(A1MPC_EINVAL, "null argument");
  const bool want_t = t_rel || t_abs || t_world;
  if (want_t && (!lin_vel || !lin_vel_d || !rot_z || !rot || !root_pos)) return fail(A1MPC_EINVAL, "foothold targets need lin_vel, lin_vel_d, rot_z, rot, root_pos");
  if (B <= 0 || gp->horizon < 0 || gp->horizon > A1MPC_MAX_HORIZON) return fail(A1MPC_EINVAL, "bad B or horizon");
  CK(cudaSetDevice(h->device));
  GaitDev G;
  G.cpg = gp->counter_per_gait; G.cps = gp->counter_per_swing; G.cdt = gp->control_dt; G.dxl = gp->foot_delta_x_limit; G.dyl = gp->foot_delta_y_limit;
  for (int i = 0; i < 12; ++i) G.dfp[i] = gp->default_foot_pos[i];
  G.N = gp->horizon;
  Stage st(h, B);
  st.inout(gait_counter, 4); st.in(gait_counter_speed, 4); st.in(movement_mode, 1);
  if (want_t) {   // the kernel reads the foothold inputs only for the foothold outputs
    st.in(lin_vel, 3); st.in(lin_vel_d, 3); st.in(rot_z, 9); st.in(rot, 9); st.in(root_pos, 3);
  } else {
    for (const void* p : {lin_vel, lin_vel_d, rot_z, rot, root_pos}) st.unused(p);
  }
  st.out(plan_contacts, 1); st.out(contact_sched, G.N); st.out(t_rel, 12); st.out(t_abs, 12); st.out(t_world, 12);
  int rc;
  if ((rc = st.begin())) return rc;
  update_plan_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, G, gait_counter, gait_counter_speed, movement_mode, lin_vel, lin_vel_d, rot_z, rot,
                                                              root_pos, plan_contacts, contact_sched, t_rel, t_abs, t_world);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_gait_row(int gait_type, double row[6]) {
  if (!row) return fail(A1MPC_EINVAL, "null argument");
  // offsets FL FR RL RR, counter_per_gait, counter_per_swing; the trot is A1CtrlStates.h:24-25, 322-326
  static const double rows[5][6] = {{0, 120, 120, 0, 240, 120},    // trot: diagonal pairs
                                    {0, 120, 0, 120, 240, 120},    // pace: lateral pairs
                                    {0, 0, 120, 120, 240, 120},    // bound: front pair, rear pair
                                    {0, 0, 0, 0, 240, 120},        // pronk: all four
                                    {120, 0, 180, 60, 240, 180}};  // lateral-sequence walk RL, FL, RR, FR, one foot in swing at a time
  if (gait_type < A1MPC_GAIT_TROT || gait_type > A1MPC_GAIT_WALK) return fail(A1MPC_EINVAL, "unknown gait type");
  for (int k = 0; k < 6; ++k) row[k] = rows[gait_type - A1MPC_GAIT_TROT][k];
  return A1MPC_OK;
}

int a1mpc_update_plan_gait_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* gait, double* gait_counter,
                                 const double* gait_counter_speed, const uint32_t* movement_mode, const double* lin_vel, const double* lin_vel_d,
                                 const double* rot_z, const double* rot, const double* root_pos, uint32_t* plan_contacts, uint32_t* contact_sched,
                                 double* t_rel, double* t_abs, double* t_world) {
  if (!h || !gp || !gait || !gait_counter || !gait_counter_speed || !movement_mode || !plan_contacts) return fail(A1MPC_EINVAL, "null argument");
  const bool want_t = t_rel || t_abs || t_world;
  if (want_t && (!lin_vel || !lin_vel_d || !rot_z || !rot || !root_pos)) return fail(A1MPC_EINVAL, "foothold targets need lin_vel, lin_vel_d, rot_z, rot, root_pos");
  if (B <= 0 || gp->horizon < 0 || gp->horizon > A1MPC_MAX_HORIZON) return fail(A1MPC_EINVAL, "bad B or horizon");
  CK(cudaSetDevice(h->device));
  GaitDev G;
  G.cpg = gp->counter_per_gait; G.cps = gp->counter_per_swing; G.cdt = gp->control_dt; G.dxl = gp->foot_delta_x_limit; G.dyl = gp->foot_delta_y_limit;
  for (int i = 0; i < 12; ++i) G.dfp[i] = gp->default_foot_pos[i];
  G.N = gp->horizon;
  Stage st(h, B);
  st.in(gait, 6); st.inout(gait_counter, 4); st.in(gait_counter_speed, 4); st.in(movement_mode, 1);
  if (want_t) {
    st.in(lin_vel, 3); st.in(lin_vel_d, 3); st.in(rot_z, 9); st.in(rot, 9); st.in(root_pos, 3);
  } else {
    for (const void* p : {lin_vel, lin_vel_d, rot_z, rot, root_pos}) st.unused(p);
  }
  st.out(plan_contacts, 1); st.out(contact_sched, G.N); st.out(t_rel, 12); st.out(t_abs, 12); st.out(t_world, 12);
  int rc;
  if ((rc = st.begin())) return rc;
  update_plan_gait_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, G, gait, gait_counter, gait_counter_speed, movement_mode, lin_vel, lin_vel_d,
                                                                   rot_z, rot, root_pos, plan_contacts, contact_sched, t_rel, t_abs, t_world);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

// ---- upstream producers of the path's inputs (SURVEY 8f.4) ---------------------------------------------------

int a1mpc_leg_kinematics_batch(a1mpc_handle* h, int B, const double* joint_pos, const double* joint_vel, const double* rot,
                               const double* rho_opt, const double* rho_fix, double* foot_pos_rel, double* jac, double* foot_vel_rel,
                               double* foot_pos_abs, double* foot_vel_abs) {
  if (!h || !joint_pos || !rho_opt || !rho_fix) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if ((foot_vel_rel || foot_vel_abs) && !joint_vel) return fail(A1MPC_EINVAL, "foot velocities need joint_vel");
  if ((foot_pos_abs || foot_vel_abs) && !rot) return fail(A1MPC_EINVAL, "body-aligned outputs need rot");
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(joint_pos, 12); st.in(joint_vel, 12); st.in(rot, 9);
  st.out(foot_pos_rel, 12); st.out(jac, 36); st.out(foot_vel_rel, 12); st.out(foot_pos_abs, 12); st.out(foot_vel_abs, 12);
  st.host_param(rho_opt, "rho_opt"); st.host_param(rho_fix, "rho_fix");
  int rc;
  if ((rc = st.begin())) return rc;
  LegParams P;
  for (int i = 0; i < 12; ++i) P.rho_opt[i] = rho_opt[i];
  for (int i = 0; i < 20; ++i) P.rho_fix[i] = rho_fix[i];
  leg_kinematics_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, joint_pos, joint_vel, rot, P, foot_pos_rel, jac, foot_vel_rel, foot_pos_abs, foot_vel_abs);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

size_t a1mpc_ekf_bytes(int B) { return B > 0 ? (size_t)B * EKF_STATE_DOUBLES * sizeof(double) : 0; }

int a1mpc_ekf_init_batch(a1mpc_handle* h, int B, void* ekf_state, const double* foot_pos_rel, const double* rot) {
  if (!h || !ekf_state || !foot_pos_rel || !rot) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(ekf_state)) return fail(A1MPC_EINVAL, "ekf_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(foot_pos_rel, 12); st.in(rot, 9);
  int rc;
  if ((rc = st.begin())) return rc;
  ekf_init_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, static_cast<double*>(ekf_state), foot_pos_rel, rot);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_ekf_update_batch(a1mpc_handle* h, int B, void* ekf_state, double dt, int assume_flat_ground, const uint32_t* movement_mode,
                           const double* imu_acc, const double* imu_ang_vel, const double* rot, const double* foot_pos_rel,
                           const double* foot_vel_rel, const double* foot_force, double* root_pos, double* root_lin_vel,
                           uint32_t* estimated_contacts, int32_t* status) {
  if (!h || !ekf_state || !movement_mode || !imu_acc || !imu_ang_vel || !rot || !foot_pos_rel || !foot_vel_rel || !foot_force)
    return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!(dt > 0.0)) return fail(A1MPC_EINVAL, "dt must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(ekf_state)) return fail(A1MPC_EINVAL, "ekf_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(movement_mode, 1); st.in(imu_acc, 3); st.in(imu_ang_vel, 3); st.in(rot, 9); st.in(foot_pos_rel, 12); st.in(foot_vel_rel, 12);
  st.in(foot_force, 4);
  st.out(root_pos, 3); st.out(root_lin_vel, 3); st.out(estimated_contacts, 1); st.out(status, 1);
  int rc;
  if ((rc = st.begin())) return rc;
  if ((rc = enqueue_ekf_update(h, B, static_cast<double*>(ekf_state), EkfParams{dt, assume_flat_ground ? 1 : 0}, movement_mode, imu_acc, imu_ang_vel, rot,
                               foot_pos_rel, foot_vel_rel, foot_force, root_pos, root_lin_vel, estimated_contacts, status)))
    return rc;
  return st.finish();
}

// ---- swing-leg control and terrain pitch (generate_swing_legs_ctrl, compute_grf's terrain adaptation) --------------------------
size_t a1mpc_swing_bytes(int B) { return B > 0 ? (size_t)B * SW_FIELDS * sizeof(double) : 0; }

int a1mpc_swing_init_batch(a1mpc_handle* h, int B, void* swing_state) {
  if (!h || !swing_state) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  swing_init_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, static_cast<double*>(swing_state));
  h->launches++;
  CK(cudaGetLastError());
  return A1MPC_OK;
}

int a1mpc_swing_legs_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* kp_foot, const double* kd_foot, void* swing_state,
                           double dt, const double* gait_counter, const uint32_t* plan_contacts, const double* rot_z, const double* foot_pos_abs,
                           const double* foot_pos_target_rel, const double* foot_force, double* f_kin, uint32_t* contacts, double* foot_pos_cur,
                           double* foot_pos_recent_contact) {
  if (!h || !gp || !kp_foot || !kd_foot || !swing_state || !gait_counter || !plan_contacts || !rot_z || !foot_pos_abs || !foot_pos_target_rel ||
      !foot_force || !f_kin || !contacts)
    return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!(dt > 0.0) || !(gp->counter_per_swing > 0.0)) return fail(A1MPC_EINVAL, "dt and counter_per_swing must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(gait_counter, 4); st.in(plan_contacts, 1); st.in(rot_z, 9); st.in(foot_pos_abs, 12); st.in(foot_pos_target_rel, 12); st.in(foot_force, 4);
  st.out(f_kin, 12); st.out(contacts, 1); st.out(foot_pos_cur, 12); st.out(foot_pos_recent_contact, 12);
  st.host_param(kp_foot, "kp_foot"); st.host_param(kd_foot, "kd_foot");
  int rc;
  if ((rc = st.begin())) return rc;
  SwingParams P;
  P.cps = gp->counter_per_swing;
  P.dt = dt;
  for (int i = 0; i < 12; ++i) { P.kp[i] = kp_foot[i]; P.kd[i] = kd_foot[i]; }
  swing_legs_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, P, static_cast<double*>(swing_state), gait_counter, plan_contacts, rot_z, foot_pos_abs,
                                                            foot_pos_target_rel, foot_force, f_kin, contacts, foot_pos_cur, foot_pos_recent_contact);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_swing_legs_gait_batch(a1mpc_handle* h, int B, const a1mpc_gait_params* gp, const double* gait, const double* kp_foot, const double* kd_foot,
                                void* swing_state, double dt, const double* gait_counter, const uint32_t* plan_contacts, const double* rot_z,
                                const double* foot_pos_abs, const double* foot_pos_target_rel, const double* foot_force, double* f_kin, uint32_t* contacts,
                                double* foot_pos_cur, double* foot_pos_recent_contact) {
  if (!h || !gp || !gait || !kp_foot || !kd_foot || !swing_state || !gait_counter || !plan_contacts || !rot_z || !foot_pos_abs || !foot_pos_target_rel ||
      !foot_force || !f_kin || !contacts)
    return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!(dt > 0.0)) return fail(A1MPC_EINVAL, "dt must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(gait, 6); st.in(gait_counter, 4); st.in(plan_contacts, 1); st.in(rot_z, 9); st.in(foot_pos_abs, 12); st.in(foot_pos_target_rel, 12);
  st.in(foot_force, 4);
  st.out(f_kin, 12); st.out(contacts, 1); st.out(foot_pos_cur, 12); st.out(foot_pos_recent_contact, 12);
  st.host_param(kp_foot, "kp_foot"); st.host_param(kd_foot, "kd_foot");
  int rc;
  if ((rc = st.begin())) return rc;
  SwingParams P;
  P.cps = gp->counter_per_swing;   // not read: each robot's row gives its own
  P.dt = dt;
  for (int i = 0; i < 12; ++i) { P.kp[i] = kp_foot[i]; P.kd[i] = kd_foot[i]; }
  swing_legs_gait_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, P, gait, static_cast<double*>(swing_state), gait_counter, plan_contacts, rot_z,
                                                                 foot_pos_abs, foot_pos_target_rel, foot_force, f_kin, contacts, foot_pos_cur,
                                                                 foot_pos_recent_contact);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_terrain_pitch_batch(a1mpc_handle* h, int B, void* swing_state, int use_terrain_adapt, const double* root_pos, double* ref, size_t ref_ld,
                              double* terrain_pitch) {
  if (!h || !swing_state || !root_pos || (use_terrain_adapt && !ref)) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (ref && ref_ld < (size_t)B) return fail(A1MPC_EINVAL, "ref_ld must be >= B");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  // only row 1 of ref is written: on the host side it is staged as a dense row (ld 0 from the kernel's point of view)
  double* row = use_terrain_adapt ? ref + ref_ld : nullptr;
  Stage st(h, B);
  st.in(root_pos, 3);
  st.out(row, 1); st.out(terrain_pitch, 1);
  if (!use_terrain_adapt) st.unused(ref);
  int rc;
  if ((rc = st.begin())) return rc;
  double* kref = st.host() ? row : ref;
  const size_t kld = st.host() ? 0 : ref_ld;
  terrain_pitch_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, static_cast<double*>(swing_state), use_terrain_adapt ? 1 : 0, root_pos, kref, kld,
                                                               terrain_pitch);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_terrain_normals_batch(a1mpc_handle* h, int B, void* swing_state, int use_terrain_adapt, const double* root_pos, double* ref, size_t ref_ld,
                                double* terrain_pitch, double* normals) {
  if (!h || !swing_state || !root_pos || !normals || (use_terrain_adapt && !ref)) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (ref && ref_ld < (size_t)B) return fail(A1MPC_EINVAL, "ref_ld must be >= B");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  double* row = use_terrain_adapt ? ref + ref_ld : nullptr;   // as in a1mpc_terrain_pitch_batch
  Stage st(h, B);
  st.in(root_pos, 3);
  st.out(row, 1); st.out(terrain_pitch, 1); st.out(normals, 12);
  if (!use_terrain_adapt) st.unused(ref);
  int rc;
  if ((rc = st.begin())) return rc;
  double* kref = st.host() ? row : ref;
  const size_t kld = st.host() ? 0 : ref_ld;
  terrain_normals_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, static_cast<double*>(swing_state), use_terrain_adapt ? 1 : 0, root_pos, kref,
                                                                 kld, terrain_pitch, normals, nullptr, nullptr, 0);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_surface_normals_batch(a1mpc_handle* h, int B, const void* swing_state, const double* root_pos, double* normals) {
  if (!h || !swing_state || !root_pos || !normals) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(swing_state)) return fail(A1MPC_EINVAL, "swing_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(root_pos, 3);
  st.out(normals, 12);
  int rc;
  if ((rc = st.begin())) return rc;
  surface_normals_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, static_cast<const double*>(swing_state), root_pos, normals);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

// ---- orientation and command stages (the adapters' IMU / pose callbacks and main_update's front half) ------------------------
size_t a1mpc_imu_bytes(int B) { return B > 0 ? (size_t)B * imu_state_doubles() * sizeof(double) : 0; }

int a1mpc_plan_forces_batch(a1mpc_handle* h, int B, const double* rot, const double* u_full, const uint32_t* step, double* f_body) {
  if (!h || !rot || !u_full || !step || !f_body) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  const int N = h->cfg.horizon;
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(rot, 9); st.in(u_full, 12 * (size_t)N); st.in(step, 1); st.inout(f_body, 12);
  int rc;
  if ((rc = st.begin())) return rc;
  plan_forces_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, N, rot, u_full, step, f_body);
  h->launches++;
  CK(cudaGetLastError());
  return st.finish();
}

int a1mpc_imu_init_batch(a1mpc_handle* h, int B, void* imu_state) {
  if (!h || !imu_state) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(imu_state)) return fail(A1MPC_EINVAL, "imu_state must be device memory (a1mpc_device_alloc)");
  CK(imu_init_launch(B, static_cast<double*>(imu_state), h->stream));
  h->launches++;
  return A1MPC_OK;
}

int a1mpc_orientation_batch(a1mpc_handle* h, int B, const double* quat, const double* gyro, const double* acc, void* imu_state, double* rot,
                            double* rot_z, double* x0, size_t ld, double* imu_acc, double* imu_ang_vel) {
  if (!h || !quat || !gyro) return fail(A1MPC_EINVAL, "null argument");
  if (imu_acc && !acc) return fail(A1MPC_EINVAL, "imu_acc needs acc");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (ld < (size_t)B) return fail(A1MPC_EINVAL, "ld < B");
  CK(cudaSetDevice(h->device));
  if (imu_state && !is_device_ptr(imu_state)) return fail(A1MPC_EINVAL, "imu_state must be device memory (a1mpc_device_alloc)");
  // x0 rows 0-2 (root_euler) and 6-8 (root_ang_vel) are two arrays: the rows in between belong to the estimator
  double* euler = x0;
  double* ang_vel = x0 ? x0 + 6 * ld : nullptr;
  Stage st(h, B);
  st.in(quat, 4); st.in(gyro, 3); st.in(acc, 3);
  st.out(rot, 9, 8, ld); st.out(rot_z, 9, 8, ld); st.out(euler, 3, 8, ld); st.out(ang_vel, 3, 8, ld);
  st.out(imu_acc, 3); st.out(imu_ang_vel, 3);
  int rc;
  if ((rc = st.begin())) return rc;
  const size_t kld = st.host() ? (size_t)B : ld;
  CK(orientation_launch(B, quat, gyro, acc, static_cast<double*>(imu_state), rot, rot_z, euler, ang_vel, kld, imu_acc, imu_ang_vel, h->stream));
  h->launches++;
  return st.finish();
}

size_t a1mpc_command_bytes(int B) { return B > 0 ? (size_t)B * command_state_doubles() * sizeof(double) : 0; }

int a1mpc_command_init_batch(a1mpc_handle* h, int B, void* cmd_state, const a1mpc_command_params* cp, double* ref, size_t ref_ld) {
  if (!h || !cmd_state || !cp) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (ref && ref_ld < (size_t)B) return fail(A1MPC_EINVAL, "ref_ld must be >= B");
  if (cp->variant != A1MPC_VARIANT_GAZEBO && cp->variant != A1MPC_VARIANT_HARDWARE && cp->variant != A1MPC_VARIANT_ISAAC)
    return fail(A1MPC_EINVAL, "unknown variant");
  if (!(cp->body_height_min <= cp->body_height_max)) return fail(A1MPC_EINVAL, "body_height_min must not exceed body_height_max");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(cmd_state)) return fail(A1MPC_EINVAL, "cmd_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.out(ref, 9, 8, ref_ld);
  int rc;
  if ((rc = st.begin())) return rc;
  CK(command_init_launch(B, *cp, static_cast<double*>(cmd_state), ref, st.host() ? (size_t)B : ref_ld, h->stream));
  h->launches++;
  return st.finish();
}

int a1mpc_command_batch(a1mpc_handle* h, int B, void* cmd_state, double dt, const double* cmd, const double* root_pos, size_t root_pos_ld,
                        uint32_t* movement_mode, double* kp_linear, double* ref, size_t ref_ld, double* des, size_t stance_ld) {
  if (!h || !cmd_state || !cmd || !root_pos || !movement_mode || !kp_linear) return fail(A1MPC_EINVAL, "null argument");
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (!(dt > 0.0)) return fail(A1MPC_EINVAL, "dt must be positive");
  if (root_pos_ld < (size_t)B || stance_ld < (size_t)B || (ref && ref_ld < (size_t)B)) return fail(A1MPC_EINVAL, "ld < B");
  CK(cudaSetDevice(h->device));
  if (!is_device_ptr(cmd_state)) return fail(A1MPC_EINVAL, "cmd_state must be device memory (a1mpc_device_alloc)");
  Stage st(h, B);
  st.in(cmd, 7); st.in(root_pos, 3, 8, root_pos_ld);
  st.out(movement_mode, 1); st.out(kp_linear, 3, 8, stance_ld); st.inout(ref, 9, 8, ref_ld); st.out(des, 12, 8, stance_ld);
  int rc;
  if ((rc = st.begin())) return rc;
  const bool hm = st.host();
  CK(command_launch(B, dt, static_cast<double*>(cmd_state), cmd, root_pos, hm ? (size_t)B : root_pos_ld, movement_mode, kp_linear, ref,
                    hm ? (size_t)B : ref_ld, des, hm ? (size_t)B : stance_ld, h->stream));
  h->launches++;
  return st.finish();
}

// ---- a whole control tick (a1mpc_tick_*) ---------------------------------------------------------------------------------------
}  // extern "C"

struct a1mpc_tick {
  a1mpc_handle* h = nullptr;
  int B = 0;
  a1mpc_tick_params tp;
  bool first = true;      // the next run initialises the EKF instead of updating it
  bool pending = false;   // a partial reset has flagged robots in `reset` whose EKF the next run initialises
  void* mem = nullptr;    // one device allocation holding everything below
  // intermediates, dense [rows][B]
  double *rot, *rz, *x0, *ia, *ig, *fpr, *fvr, *jac, *foot, *kpl, *des, *ref, *fk, *f_body;
  uint32_t *mode, *contact, *est_contacts;
  uint32_t* sched;        // the scheduled tick's contact schedule [N][B] (gait.horizon = N), else NULL
  int32_t *status, *est_status;
  // state
  double *gc, *tau, *imu, *cmd, *swing, *ekf;
  uint32_t* warm;
  uint8_t* reset;         // [B]: robot reset by a1mpc_tick_reset_robots since the last run (ekf_init_pending)
  // the friction pyramids of the solve (a1mpc_tick_set_terrain) or of the stance QP (a1mpc_tick_set_stance_terrain)
  int terrain = A1MPC_TERRAIN_FLAT;
  const double* given = nullptr;   // A1MPC_TERRAIN_GIVEN: the caller's normals [12][B]
  void* tmem = nullptr;            // allocated by the first set_terrain / set_stance_terrain to a non-flat source: normals, then held
  double* normals = nullptr;       // [12][B] terrain_normals_kernel's (MPC) or surface_normals_kernel's (QP) estimate
  uint32_t* held = nullptr;        // [N][B] the held pattern as a schedule (gait.horizon = 0), else NULL
  // the MPC period (a1mpc_tick_set_mpc_period); rmem and plan are allocated by the first call that needs them
  int period = 1;
  int playback = A1MPC_PLAYBACK_HOLD;
  void* rmem = nullptr;            // runs [B] (n_b), then since [B] (j_b)
  uint32_t *runs = nullptr, *since = nullptr;
  double* plan = nullptr;          // [12 N][B] each robot's u_full of its last solve (A1MPC_PLAYBACK_PLAN)
  // per-robot gaits (a1mpc_tick_set_gaits); gmem is allocated by the first call with rows
  void* gmem = nullptr;            // gait [6][B], then the row check's result word
  double* gait = nullptr;
  unsigned long long* gbad = nullptr;
  bool gaits = false;              // the front runs its gait twin on `gait`
};

namespace {

int tick_reset_impl(a1mpc_tick* t) {
  a1mpc_handle* h = t->h;
  const int B = t->B;
  const size_t lb = (size_t)B;
  CK(cudaSetDevice(h->device));
  CK(cudaMemsetAsync(t->x0, 0, 12 * lb * sizeof(double), h->stream));
  CK(cudaMemsetAsync(t->gc, 0, 4 * lb * sizeof(double), h->stream));
  CK(cudaMemsetAsync(t->tau, 0, 12 * lb * sizeof(double), h->stream));
  if (t->imu) {
    CK(imu_init_launch(B, t->imu, h->stream));
    h->launches++;
  }
  const bool mpc = t->tp.mode == A1MPC_TICK_MPC;
  CK(command_init_launch(B, t->tp.command, t->cmd, mpc ? t->ref : nullptr, lb, h->stream));
  swing_init_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->swing);
  h->launches += 2;
  CK(cudaGetLastError());
  if (t->warm) CK(cudaMemsetAsync(t->warm, 0, a1mpc_warm_bytes(h, B), h->stream));
  CK(cudaMemsetAsync(t->reset, 0, lb, h->stream));   // the EKF init of every robot supersedes a pending partial one
  if (t->rmem) CK(cudaMemsetAsync(t->rmem, 0, 2 * lb * sizeof(uint32_t), h->stream));   // every robot solves on the next run
  t->first = true;
  t->pending = false;
  return A1MPC_OK;
}

// the first non-flat terrain source of a tick: its normals [12][B] and, held_bytes > 0, the held pattern as a schedule
int tick_terrain_alloc(a1mpc_tick* t, size_t held_bytes) {
  if (t->tmem) return A1MPC_OK;
  auto pad = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t nb = pad(12 * (size_t)t->B * sizeof(double));
  if (cudaMalloc(&t->tmem, nb + held_bytes) != cudaSuccess) {
    cudaGetLastError();
    t->tmem = nullptr;
    return fail(A1MPC_ENOMEM, "cudaMalloc failed");
  }
  t->normals = static_cast<double*>(t->tmem);
  t->held = held_bytes ? reinterpret_cast<uint32_t*>(static_cast<char*>(t->tmem) + nb) : nullptr;
  return A1MPC_OK;
}

}  // namespace

extern "C" {

int a1mpc_default_tick_params(int variant, int mode, a1mpc_tick_params* tp) {
  if (!tp) return fail(A1MPC_EINVAL, "null argument");
  if (variant != A1MPC_VARIANT_GAZEBO && variant != A1MPC_VARIANT_HARDWARE && variant != A1MPC_VARIANT_ISAAC) return fail(A1MPC_EINVAL, "unknown variant");
  if (mode != A1MPC_TICK_QP && mode != A1MPC_TICK_MPC) return fail(A1MPC_EINVAL, "unknown mode");
  std::memset(tp, 0, sizeof(*tp));
  const bool mpc = mode == A1MPC_TICK_MPC;
  const int v = variant;   // 0 Gazebo, 1 hardware, 2 Isaac
  tp->mode = mode;
  // use_terrain_adapt: A1CtrlStates.h:137 (ROS default 1); isaac_a1_mpc.yaml:3 sets 0
  tp->use_terrain_adapt = (v == A1MPC_VARIANT_ISAAC && mpc) ? 0 : 1;
  // every adapter constructs A1BasicEKF a1_estimate (GazeboA1ROS.h:157, HardwareA1ROS.h:134, IsaacA1ROS.h:107): assume_flat_ground = true
  // (A1BasicEKF.cpp:40)
  tp->assume_flat_ground = 1;
  // gait: counter_per_gait / _swing (A1CtrlStates.h:24-25), control_dt = MAIN_UPDATE_FREQUENCY / 1000 (A1CtrlStates.h:332, A1Params.h:11),
  // FOOT_DELTA_{X,Y}_LIMIT (A1Params.h:44-45); default_foot_pos 3 x 4 row-major (x, y, z rows; FL, FR, RL, RR) from
  // config/<variant>_a1_<mode>.yaml a1_default_foot_pos_* (gazebo_a1_mpc.yaml:17-31, gazebo_a1_qp.yaml:10-24, hardware_a1_mpc.yaml:18-32,
  // hardware_a1_qp.yaml:11-25, isaac_a1_mpc.yaml:18-32, isaac_a1_qp.yaml:10-24)
  tp->gait.counter_per_gait = 240.0;
  tp->gait.counter_per_swing = 120.0;
  tp->gait.control_dt = 2.5 / 1000.0;
  tp->gait.foot_delta_x_limit = 0.1;
  tp->gait.foot_delta_y_limit = 0.1;
  tp->gait.horizon = 0;
  {
    const double front_x = v == A1MPC_VARIANT_ISAAC ? (mpc ? 0.24 : 0.25) : 0.17;
    const double z = v == A1MPC_VARIANT_HARDWARE ? (mpc ? -0.3 : -0.33) : (v == A1MPC_VARIANT_ISAAC ? (mpc ? -0.35 : -0.33) : -0.35);
    const double fp[12] = {front_x, front_x, -0.17, -0.17, 0.15, -0.15, 0.15, -0.15, z, z, z, z};
    for (int i = 0; i < 12; ++i) tp->gait.default_foot_pos[i] = fp[i];
  }
  // command: the adapter's initial joy_cmd_body_height (GazeboA1ROS.h:130, HardwareA1ROS.h:107, IsaacA1ROS.h:80), JOY_CMD_BODY_HEIGHT_MIN /
  // _MAX (A1Params.h:16-17); kp_linear = a1_kp_linear_* (A1CtrlStates.h:273-275, ROS defaults 120, 120, 500; the QP configs set them:
  // gazebo_a1_qp.yaml:54-56, hardware_a1_qp.yaml:55-57, isaac_a1_qp.yaml:54-56) and kp_linear_lock = its x and y (A1CtrlStates.h:298-299)
  tp->command.variant = variant;
  tp->command.body_height = v == A1MPC_VARIANT_GAZEBO ? 0.3 : (v == A1MPC_VARIANT_HARDWARE ? 0.12 : 0.32);
  tp->command.body_height_min = 0.1;
  tp->command.body_height_max = 0.32;
  {
    static const double kpl_qp[3][3] = {{100.0, 100.0, 300.0}, {400.0, 400.0, 1500.0}, {1450.0, 1450.0, 3800.0}};
    const double kpl_ros[3] = {120.0, 120.0, 500.0};
    const double* kpl = mpc ? kpl_ros : kpl_qp[v];
    for (int i = 0; i < 3; ++i) tp->command.kp_linear[i] = kpl[i];
    tp->command.kp_linear_lock[0] = kpl[0];
    tp->command.kp_linear_lock[1] = kpl[1];
  }
  // leg geometry (GazeboA1ROS.cpp:75-97, HardwareA1ROS.cpp:52-74, IsaacA1ROS.cpp:38-60): rho_opt = 0; rho_fix = leg_offset_x, leg_offset_y,
  // motor_offset, upper_leg_length (0.21 Gazebo, 0.20 hardware, 0.22 Isaac), lower_leg_length (LOWER_LEG_LENGTH = 0.21, A1Params.h:36;
  // 0.20 hardware)
  {
    const double upper = v == A1MPC_VARIANT_GAZEBO ? 0.21 : (v == A1MPC_VARIANT_HARDWARE ? 0.20 : 0.22);
    const double lower = v == A1MPC_VARIANT_HARDWARE ? 0.20 : 0.21;
    const double ox[4] = {0.1805, 0.1805, -0.1805, -0.1805}, oy[4] = {0.047, -0.047, 0.047, -0.047}, mo[4] = {0.0838, -0.0838, 0.0838, -0.0838};
    for (int i = 0; i < 4; ++i) {
      const double r[5] = {ox[i], oy[i], mo[i], upper, lower};
      for (int k = 0; k < 5; ++k) tp->rho_fix[5 * i + k] = r[k];
    }
  }
  // swing-leg and torque gains: a1_kp_foot_*, a1_kd_foot_*, a1_km_foot_* of config/<variant>_a1_<mode>.yaml (gazebo_a1_mpc.yaml:77-87,
  // gazebo_a1_qp.yaml:34-44, hardware_a1_mpc.yaml:78-88, hardware_a1_qp.yaml:35-45, isaac_a1_mpc.yaml:78-88, isaac_a1_qp.yaml:34-44);
  // torques_gravity (A1CtrlStates.h:129)
  {
    // [variant][mode QP, MPC][kp x y z, kd x y z, km x y z]
    static const double g[3][2][9] = {{{300, 400, 400, 8, 8, 8, 0.1, 0.1, 0.1}, {200, 200, 150, 10, 10, 5, 0.1, 0.1, 0.1}},
                                      {{260, 260, 350, 6, 6, 5, 0.1, 0.1, 0.1}, {120, 120, 80, 6, 6, 5, 0.1, 0.1, 0.1}},
                                      {{4250, 4250, 3000, 0, 0, 0, 0.5, 0.5, 0.5}, {3250, 3250, 4000, 5, 5, 5, 0.5, 0.5, 0.5}}};
    const double* k = g[v][mpc ? 1 : 0];
    for (int i = 0; i < 12; ++i) { tp->kp_foot[i] = k[i % 3]; tp->kd_foot[i] = k[3 + i % 3]; }
    for (int a = 0; a < 3; ++a) tp->km_foot[a] = k[6 + a];
    const double tg[12] = {0.80, 0, 0, -0.80, 0, 0, 0.80, 0, 0, -0.80, 0, 0};
    for (int i = 0; i < 12; ++i) tp->torques_gravity[i] = tg[i];
  }
  // the stance PD gains of the QP branch: a1_kd_linear_*, a1_kp_angular_*, a1_kd_angular_* (gazebo_a1_qp.yaml:58-68, hardware_a1_qp.yaml:59-69,
  // isaac_a1_qp.yaml:58-68); the MPC configs set none, so MPC mode gets the ROS defaults (A1CtrlStates.h:278-296: 70, 70, 120 / 250, 35, 1 /
  // 1.5, 1.5, 30), which the MPC branch does not read
  {
    static const double qp[3][9] = {{70, 70, 120, 150, 150, 1, 4.5, 4.5, 30},
                                    {300, 200, 120, 40, 40, 10, 1, 1, 0.5},
                                    {2600, 2600, 0, 420, 420, 150, 0, 0, 560}};
    static const double ros[9] = {70, 70, 120, 250, 35, 1, 1.5, 1.5, 30};
    const double* k = mpc ? ros : qp[v];
    for (int a = 0; a < 3; ++a) { tp->kd_linear[a] = k[a]; tp->kp_angular[a] = k[3 + a]; tp->kd_angular[a] = k[6 + a]; }
  }
  return A1MPC_OK;
}

int a1mpc_tick_create(a1mpc_handle* h, int B, const a1mpc_tick_params* tp, a1mpc_tick** out) {
  if (!h || !tp || !out) return fail(A1MPC_EINVAL, "null argument");
  *out = nullptr;
  if (B <= 0) return fail(A1MPC_EINVAL, "B must be positive");
  if (h->cfg.precision != 64) return fail(A1MPC_EINVAL, "a tick needs precision 64 (its front stages are fp64)");
  if (tp->mode != A1MPC_TICK_QP && tp->mode != A1MPC_TICK_MPC) return fail(A1MPC_EINVAL, "unknown mode");
  const int v = tp->command.variant;
  if (v != A1MPC_VARIANT_GAZEBO && v != A1MPC_VARIANT_HARDWARE && v != A1MPC_VARIANT_ISAAC) return fail(A1MPC_EINVAL, "unknown variant");
  if (!(tp->gait.counter_per_swing > 0.0)) return fail(A1MPC_EINVAL, "counter_per_swing must be positive");
  if (!(tp->command.body_height_min <= tp->command.body_height_max)) return fail(A1MPC_EINVAL, "body_height_min must not exceed body_height_max");
  const bool mpc = tp->mode == A1MPC_TICK_MPC;
  if (mpc && tp->gait.horizon != 0 && tp->gait.horizon != h->cfg.horizon)
    return fail(A1MPC_EINVAL, "gait.horizon must be 0 (the held contact pattern) or the handle's horizon (the scheduled tick)");
  const bool sched = mpc && tp->gait.horizon != 0;
  CK(cudaSetDevice(h->device));
  const size_t lb = (size_t)B;
  const bool warm = mpc && h->cfg.horizon == 10;
  const bool filtered = v != A1MPC_VARIANT_HARDWARE;
  auto pad = [](size_t b) { return (b + 255) & ~(size_t)255; };
  // [rows][B] doubles of every intermediate and state array, then the 4-byte arrays, the schedule and the warm buffer
  const size_t nd[] = {9, 9, 12, 3, 3, 12, 12, 36, 12, 3, 12, 9, 12, 12, 4, 12, filtered ? imu_state_doubles() : 0, command_state_doubles(),
                       (size_t)SW_FIELDS, (size_t)EKF_STATE_DOUBLES};
  size_t bytes = 0;
  for (size_t r : nd) bytes += pad(r * lb * sizeof(double));
  bytes += 5 * pad(lb * 4);
  if (sched) bytes += pad((size_t)h->cfg.horizon * lb * 4);
  if (warm) bytes += pad(a1mpc_warm_bytes(h, B));
  bytes += pad(lb);
  a1mpc_tick* t = new a1mpc_tick();
  t->h = h; t->B = B; t->tp = *tp;
  if (cudaMalloc(&t->mem, bytes) != cudaSuccess) {
    cudaGetLastError();
    delete t;
    return fail(A1MPC_ENOMEM, "cudaMalloc failed");
  }
  char* cur = static_cast<char*>(t->mem);
  auto take = [&](size_t n) { char* p = n ? cur : nullptr; cur += pad(n); return p; };
  double** dst[] = {&t->rot, &t->rz, &t->x0, &t->ia, &t->ig, &t->fpr, &t->fvr, &t->jac, &t->foot, &t->kpl, &t->des, &t->ref, &t->fk, &t->f_body,
                    &t->gc, &t->tau, &t->imu, &t->cmd, &t->swing, &t->ekf};
  for (size_t i = 0; i < sizeof(nd) / sizeof(nd[0]); ++i) *dst[i] = reinterpret_cast<double*>(take(nd[i] * lb * sizeof(double)));
  t->mode = reinterpret_cast<uint32_t*>(take(lb * 4));
  t->contact = reinterpret_cast<uint32_t*>(take(lb * 4));
  t->est_contacts = reinterpret_cast<uint32_t*>(take(lb * 4));
  t->status = reinterpret_cast<int32_t*>(take(lb * 4));
  t->est_status = reinterpret_cast<int32_t*>(take(lb * 4));
  t->sched = sched ? reinterpret_cast<uint32_t*>(take((size_t)h->cfg.horizon * lb * 4)) : nullptr;
  t->warm = warm ? reinterpret_cast<uint32_t*>(take(a1mpc_warm_bytes(h, B))) : nullptr;
  t->reset = reinterpret_cast<uint8_t*>(take(lb));
  int rc;
  // the scheduled solve's record queues too, so that a run allocates nothing
  if ((rc = ensure_capacity(h, B)) || (sched && (rc = ensure_capacity_ext(h, B))) || (rc = ensure_lists(h, stance_scratch_bytes(B))) ||
      (rc = tick_reset_impl(t))) {
    a1mpc_tick_destroy(t);
    return rc;
  }
  *out = t;
  return A1MPC_OK;
}

int a1mpc_tick_reset(a1mpc_tick* t) {
  if (!t) return fail(A1MPC_EINVAL, "null argument");
  return tick_reset_impl(t);
}

int a1mpc_tick_reset_robots(a1mpc_tick* t, const uint8_t* mask) {
  if (!t || !mask) return fail(A1MPC_EINVAL, "null argument");
  a1mpc_handle* h = t->h;
  const int B = t->B;
  CK(cudaSetDevice(h->device));
  Stage st(h, B);
  st.in(mask, 1);
  int rc;
  if ((rc = st.begin())) return rc;
  // before the first run after create or reset every robot's EKF is initialised anyway: no flags then
  const bool flag = !t->first;
  tick_reset_robots_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, mask, command_init_params(t->tp.command), t->x0, t->gc, t->tau, t->imu, t->cmd,
                                                                    t->tp.mode == A1MPC_TICK_MPC ? t->ref : nullptr, t->swing, t->warm,
                                                                    WARM_HDR + 4 * h->cfg.horizon, flag ? t->reset : nullptr);
  h->launches++;
  if (t->rmem) {   // a period > 1 has been set: the masked robots solve on their next run
    tick_rate_reset_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, mask, t->runs, t->since);
    h->launches++;
  }
  CK(cudaGetLastError());
  t->pending = t->pending || flag;
  return st.finish();
}

int a1mpc_tick_set_terrain(a1mpc_tick* t, int source, const double* normals) {
  if (!t) return fail(A1MPC_EINVAL, "null argument");
  if (source != A1MPC_TERRAIN_FLAT && source != A1MPC_TERRAIN_ESTIMATED && source != A1MPC_TERRAIN_GIVEN) return fail(A1MPC_EINVAL, "unknown terrain source");
  if (source == A1MPC_TERRAIN_FLAT) {
    t->terrain = source;
    t->given = nullptr;
    return A1MPC_OK;
  }
  a1mpc_handle* h = t->h;
  if (t->tp.mode != A1MPC_TICK_MPC) return fail(A1MPC_EINVAL, "terrain normals need MPC mode (the stance QP keeps its world-z pyramid)");
  for (int i = 0; i < 4; ++i)
    if (h->cfg.r[3 * i] != h->cfg.r[3 * i + 1] || h->cfg.r[3 * i] != h->cfg.r[3 * i + 2])
      return fail(A1MPC_EINVAL, "terrain normals need isotropic r weights per foot (r[3i] == r[3i+1] == r[3i+2])");
  if (source == A1MPC_TERRAIN_GIVEN && !normals) return fail(A1MPC_EINVAL, "A1MPC_TERRAIN_GIVEN needs a normals array");
  CK(cudaSetDevice(h->device));
  if (source == A1MPC_TERRAIN_GIVEN && !is_device_ptr(normals)) return fail(A1MPC_EINVAL, "the given normals must be device memory");
  const size_t lb = (size_t)t->B;
  int rc;
  if ((rc = tick_terrain_alloc(t, t->sched ? 0 : (size_t)h->cfg.horizon * lb * 4))) return rc;
  if ((rc = ensure_capacity_ext(h, lb))) return rc;   // so that a run allocates nothing
  t->terrain = source;
  t->given = source == A1MPC_TERRAIN_GIVEN ? normals : nullptr;
  return A1MPC_OK;
}

int a1mpc_tick_set_stance_terrain(a1mpc_tick* t, int source, const double* normals) {
  if (!t) return fail(A1MPC_EINVAL, "null argument");
  if (t->tp.mode != A1MPC_TICK_QP) return fail(A1MPC_EINVAL, "the stance terrain is for QP mode: an MPC-mode tick takes a1mpc_tick_set_terrain");
  if (source != A1MPC_TERRAIN_FLAT && source != A1MPC_TERRAIN_ESTIMATED && source != A1MPC_TERRAIN_GIVEN) return fail(A1MPC_EINVAL, "unknown terrain source");
  if (source == A1MPC_TERRAIN_FLAT) {
    t->terrain = source;
    t->given = nullptr;
    return A1MPC_OK;
  }
  if (source == A1MPC_TERRAIN_GIVEN && !normals) return fail(A1MPC_EINVAL, "A1MPC_TERRAIN_GIVEN needs a normals array");
  CK(cudaSetDevice(t->h->device));
  if (source == A1MPC_TERRAIN_GIVEN && !is_device_ptr(normals)) return fail(A1MPC_EINVAL, "the given normals must be device memory");
  int rc;
  if ((rc = tick_terrain_alloc(t, 0))) return rc;   // the estimate only: the stance QP needs no schedule and no _ext queues
  t->terrain = source;
  t->given = source == A1MPC_TERRAIN_GIVEN ? normals : nullptr;
  return A1MPC_OK;
}

int a1mpc_tick_set_mpc_period(a1mpc_tick* t, int period, int playback) {
  if (!t) return fail(A1MPC_EINVAL, "null argument");
  if (t->tp.mode != A1MPC_TICK_MPC) return fail(A1MPC_EINVAL, "the MPC period is for MPC mode: the QP-mode stance QP runs on every run");
  a1mpc_handle* h = t->h;
  const int N = h->cfg.horizon;
  if (period < 1 || period > N) return fail(A1MPC_EINVAL, "period must run from 1 to the handle's horizon N = " + std::to_string(N));
  if (playback != A1MPC_PLAYBACK_HOLD && playback != A1MPC_PLAYBACK_PLAN) return fail(A1MPC_EINVAL, "unknown playback");
  CK(cudaSetDevice(h->device));
  const size_t lb = (size_t)t->B;
  if (period > 1 && !t->rmem) {
    if (cudaMalloc(&t->rmem, 2 * lb * sizeof(uint32_t)) != cudaSuccess) {
      cudaGetLastError();
      t->rmem = nullptr;
      return fail(A1MPC_ENOMEM, "cudaMalloc failed");
    }
    t->runs = static_cast<uint32_t*>(t->rmem);
    t->since = t->runs + lb;
  }
  if (period > 1 && playback == A1MPC_PLAYBACK_PLAN && !t->plan) {
    if (cudaMalloc(&t->plan, 12 * (size_t)N * lb * sizeof(double)) != cudaSuccess) {
      cudaGetLastError();
      t->plan = nullptr;
      return fail(A1MPC_ENOMEM, "cudaMalloc failed");
    }
  }
  // every robot solves on the next run: so the plan is written before it is read, and j_b stays below the new period
  if (t->rmem) CK(cudaMemsetAsync(t->rmem, 0, 2 * lb * sizeof(uint32_t), h->stream));
  t->period = period;
  t->playback = playback;
  return A1MPC_OK;
}

int a1mpc_tick_set_gaits(a1mpc_tick* t, const double* gait) {
  if (!t) return fail(A1MPC_EINVAL, "null argument");
  if (!gait) {   // the reference's trot: tp.gait and the trot offsets
    t->gaits = false;
    return A1MPC_OK;
  }
  a1mpc_handle* h = t->h;
  const int B = t->B;
  const size_t lb = (size_t)B;
  CK(cudaSetDevice(h->device));
  const size_t rows_bytes = (6 * lb * sizeof(double) + 255) & ~(size_t)255;
  if (!t->gmem) {
    if (cudaMalloc(&t->gmem, rows_bytes + sizeof(unsigned long long)) != cudaSuccess) {
      cudaGetLastError();
      t->gmem = nullptr;
      return fail(A1MPC_ENOMEM, "cudaMalloc failed");
    }
    t->gait = static_cast<double*>(t->gmem);
    t->gbad = reinterpret_cast<unsigned long long*>(static_cast<char*>(t->gmem) + rows_bytes);
  }
  // the rows are checked where they are (host rows in the staging slot) and copied into the tick only when every one is valid, so a
  // bad call leaves the previous gaits in force
  Stage st(h, B);
  st.in(gait, 6);
  int rc;
  if ((rc = st.begin())) return rc;
  CK(cudaMemsetAsync(t->gbad, 0xff, sizeof(unsigned long long), h->stream));
  gait_check_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, gait, t->gbad);
  h->launches++;
  CK(cudaGetLastError());
  unsigned long long bad = 0;
  CK(cudaMemcpyAsync(&bad, t->gbad, sizeof(bad), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (bad != ~0ull) {
    static const char* rule[4] = {"", "a non-finite entry", "counter_per_swing (row 5) outside (0, counter_per_gait)",
                                  "a reset offset (rows 0-3) outside [0, counter_per_gait)"};
    return fail(A1MPC_EINVAL, "gait row of robot " + std::to_string(bad >> 2) + ": " + rule[bad & 3ull]);
  }
  // the call returns with the rows in the tick: the caller may rewrite or free its array at once, from any stream
  CK(cudaMemcpyAsync(t->gait, gait, 6 * lb * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  t->gaits = true;
  return A1MPC_OK;
}

int a1mpc_tick_run(a1mpc_tick* t, double dt, const a1mpc_tick_inputs* in, const a1mpc_tick_outputs* out) {
  if (!t || !in || !out || !out->tau) return fail(A1MPC_EINVAL, "null argument");
  if (!in->quat || !in->gyro || !in->acc || !in->joint_pos || !in->joint_vel || !in->foot_force || !in->cmd || !in->gait_counter_speed)
    return fail(A1MPC_EINVAL, "null input array");
  if (!(dt > 0.0)) return fail(A1MPC_EINVAL, "dt must be positive");
  const bool mpc = t->tp.mode == A1MPC_TICK_MPC;
  if (!mpc && out->ref) return fail(A1MPC_EINVAL, "ref is an MPC-mode output: pass NULL in QP mode");
  a1mpc_handle* h = t->h;
  const int B = t->B;
  const size_t lb = (size_t)B;
  CK(cudaSetDevice(h->device));
  const double *quat = in->quat, *gyro = in->gyro, *acc = in->acc, *jp = in->joint_pos, *jv = in->joint_vel, *ff = in->foot_force, *cmd = in->cmd,
               *gcs = in->gait_counter_speed;
  Stage st(h, B);
  st.in(quat, 4); st.in(gyro, 3); st.in(acc, 3); st.in(jp, 12); st.in(jv, 12); st.in(ff, 4); st.in(cmd, 7); st.in(gcs, 4);
  for (const void* p : {(const void*)out->tau, (const void*)out->f_body, (const void*)out->status, (const void*)out->contacts,
                        (const void*)out->movement_mode, (const void*)out->x0, (const void*)out->ref})
    st.unused(p);   // written by the copies at the end
  int rc;
  if ((rc = st.begin())) return rc;
  if ((rc = ensure_capacity(h, B))) return rc;   // create sized the scratch and it only grows: no allocation here
  if (!mpc && (rc = ensure_lists(h, stance_scratch_bytes(B)))) return rc;
  if ((t->sched || (mpc && t->tmem)) && (rc = ensure_capacity_ext(h, B))) return rc;
  const a1mpc_tick_params& tp = t->tp;
  // 1-3: orientation and command
  CK(tick_front_a_launch(B, dt, quat, gyro, acc, t->imu, t->rot, t->rz, t->x0, t->ia, t->ig, t->cmd, cmd, t->mode, t->kpl, mpc ? t->ref : nullptr,
                         t->des, h->stream));
  // 2, 4, 5: kinematics, update_plan, swing legs; the scheduled tick also writes the schedule
  {
    LegParams LP;
    for (int i = 0; i < 12; ++i) LP.rho_opt[i] = tp.rho_opt[i];
    for (int i = 0; i < 20; ++i) LP.rho_fix[i] = tp.rho_fix[i];
    GaitDev G;
    G.cpg = tp.gait.counter_per_gait; G.cps = tp.gait.counter_per_swing; G.cdt = tp.gait.control_dt;
    G.dxl = tp.gait.foot_delta_x_limit; G.dyl = tp.gait.foot_delta_y_limit;
    for (int i = 0; i < 12; ++i) G.dfp[i] = tp.gait.default_foot_pos[i];
    G.N = t->sched ? h->cfg.horizon : 0;
    SwingParams SP;
    SP.cps = tp.gait.counter_per_swing;
    SP.dt = dt;
    for (int i = 0; i < 12; ++i) { SP.kp[i] = tp.kp_foot[i]; SP.kd[i] = tp.kd_foot[i]; }
    const double* lvd = mpc ? t->ref + 5 * lb : t->des + 6 * lb;
    if (t->gaits && t->sched)
      tick_front_sched_gait<<<(B + 127) / 128, 128, 0, h->stream>>>(B, LP, G, SP, t->gait, jp, jv, t->rot, t->rz, t->x0, lvd, t->mode, t->gc, gcs,
                                                                    t->swing, ff, t->fpr, t->jac, t->fvr, t->foot, t->fk, t->contact, t->sched);
    else if (t->gaits)
      tick_front_b_gait<<<(B + 127) / 128, 128, 0, h->stream>>>(B, LP, G, SP, t->gait, jp, jv, t->rot, t->rz, t->x0, lvd, t->mode, t->gc, gcs, t->swing,
                                                                ff, t->fpr, t->jac, t->fvr, t->foot, t->fk, t->contact);
    else if (t->sched)
      tick_front_sched<<<(B + 127) / 128, 128, 0, h->stream>>>(B, LP, G, SP, jp, jv, t->rot, t->rz, t->x0, lvd, t->mode, t->gc, gcs, t->swing, ff,
                                                               t->fpr, t->jac, t->fvr, t->foot, t->fk, t->contact, t->sched);
    else
      tick_front_b<<<(B + 127) / 128, 128, 0, h->stream>>>(B, LP, G, SP, jp, jv, t->rot, t->rz, t->x0, lvd, t->mode, t->gc, gcs, t->swing, ff, t->fpr,
                                                           t->jac, t->fvr, t->foot, t->fk, t->contact);
    h->launches += 2;
    CK(cudaGetLastError());
  }
  // 6: EKF into x0 rows 3-5 and 9-11
  if (t->first) {
    ekf_init_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->ekf, t->fpr, t->rot);
    h->launches++;
    CK(cudaGetLastError());
  } else if ((rc = enqueue_ekf_update(h, B, t->ekf, EkfParams{dt, tp.assume_flat_ground ? 1 : 0}, t->mode, t->ia, t->ig, t->rot, t->fpr, t->fvr, ff,
                                      t->x0 + 3 * lb, t->x0 + 9 * lb, t->est_contacts, t->est_status))) {
    return rc;
  } else if (t->pending) {
    // robots reset by a1mpc_tick_reset_robots: the init over the update, as on their first run
    ekf_init_pending<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->reset, t->ekf, t->fpr, t->rot, t->x0);
    h->launches++;
    CK(cudaGetLastError());
  }
  t->first = false;
  t->pending = false;
  // 7: terrain pitch and the MPC solve, or the stance QP.  A multi-rate tick (period > 1) solves the robots that are due this run
  // (the pack kernels skip the others), the scheduled tick with shift = period as a due robot's stored faces are `period` schedule
  // steps old; then tick_rate_kernel advances the counters and, with a plan, plays it back for the others.
  const uint32_t* runs = t->period > 1 ? t->runs : nullptr;
  double* plan = runs && t->playback == A1MPC_PLAYBACK_PLAN ? t->plan : nullptr;
  if (mpc && t->terrain != A1MPC_TERRAIN_FLAT) {
    // the same stage plus the estimated normals (and the held pattern as a schedule), then the solve of a1mpc_solve_batch_ext_warm
    // with normals: shift 1 on the scheduled tick's schedule, shift 0 on the held one (a1mpc_solve_batch_ext at horizon 20)
    terrain_normals_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->swing, tp.use_terrain_adapt ? 1 : 0, t->x0 + 3 * lb, t->ref, lb, nullptr,
                                                                   t->normals, t->contact, t->held, h->cfg.horizon);
    h->launches++;
    CK(cudaGetLastError());
    const DevInputs di{t->x0, t->rot, t->foot, t->ref, t->contact, lb, 0};
    const DevOutputs dout{t->f_body, t->status, nullptr, plan, lb, 0};
    const double* nrm = t->terrain == A1MPC_TERRAIN_GIVEN ? t->given : t->normals;
    if ((rc = t->sched ? enqueue_solve_ext(h, B, di, t->sched, nrm, dout, t->warm, t->period, runs, t->period)
                       : enqueue_solve_ext(h, B, di, t->held, nrm, dout, t->warm, 0, runs, t->period)))
      return rc;
  } else if (mpc) {
    terrain_pitch_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->swing, tp.use_terrain_adapt ? 1 : 0, t->x0 + 3 * lb, t->ref, lb, nullptr);
    h->launches++;
    CK(cudaGetLastError());
    const DevInputs di{t->x0, t->rot, t->foot, t->ref, t->contact, lb, 0};
    const DevOutputs dout{t->f_body, t->status, nullptr, plan, lb, 0};
    // held pattern: a1mpc_solve_batch_warm, shift 0 (cold at horizon 20).  Scheduled: a1mpc_solve_batch_ext_warm on the schedule with
    // world-z pyramids, shift 1 as the schedule moves one step per tick (a1mpc_solve_batch_ext at horizon 20, where t->warm is NULL)
    if ((rc = t->sched ? enqueue_solve_ext(h, B, di, t->sched, nullptr, dout, t->warm, t->period, runs, t->period)
                       : enqueue_solve(h, B, di, dout, t->warm, 0, runs, t->period)))
      return rc;
  } else {
    // a1mpc_tick_set_stance_terrain: the walking surface's normal (no terrain stage in QP mode) or the given normals, then the stance QP
    // with them; FLAT: world z
    const double* nrm = t->terrain == A1MPC_TERRAIN_GIVEN ? t->given : nullptr;
    if (t->terrain == A1MPC_TERRAIN_ESTIMATED) {
      surface_normals_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->swing, t->x0 + 3 * lb, t->normals);
      h->launches++;
      CK(cudaGetLastError());
      nrm = t->normals;
    }
    double gains[9];
    for (int i = 0; i < 3; ++i) { gains[i] = tp.kd_linear[i]; gains[3 + i] = tp.kp_angular[i]; gains[6 + i] = tp.kd_angular[i]; }
    int nl = 0;
    cudaError_t e = stance_qp_launch(h->sm_count, B, lb, t->x0, t->rot, t->rz, t->foot, t->contact, t->des, t->kpl, gains, h->cfg.mass, nrm,
                                     t->f_body, t->status, nullptr, h->d_lists, h->stream, &nl);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("stance_qp kernels: ") + cudaGetErrorString(e));
    h->launches += nl;
  }
  if (runs) {
    tick_rate_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->period, h->cfg.horizon, t->runs, t->since, t->rot, plan, t->f_body);
    h->launches++;
    CK(cudaGetLastError());
  }
  // 8: joint torques
  {
    TorqueParams P;
    for (int i = 0; i < 3; ++i) P.km[i] = tp.km_foot[i];
    for (int i = 0; i < 12; ++i) P.tg[i] = tp.torques_gravity[i];
    joint_torques_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(B, t->f_body, t->fk, t->jac, t->contact, P, t->tau);
    h->launches++;
    CK(cudaGetLastError());
  }
  const cudaMemcpyKind kind = st.host() ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  const struct { void* dst; const void* src; size_t bytes; } copies[] = {
      {out->tau, t->tau, 12 * lb * 8}, {out->f_body, t->f_body, 12 * lb * 8}, {out->status, t->status, lb * 4}, {out->contacts, t->contact, lb * 4},
      {out->movement_mode, t->mode, lb * 4}, {out->x0, t->x0, 12 * lb * 8}, {out->ref, t->ref, 9 * lb * 8}};
  for (const auto& c : copies)
    if (c.dst) CK(cudaMemcpyAsync(c.dst, c.src, c.bytes, kind, h->stream));
  return st.finish();
}

int a1mpc_tick_destroy(a1mpc_tick* t) {
  if (!t) return A1MPC_OK;
  cudaSetDevice(t->h->device);
  cudaStreamSynchronize(t->h->stream);
  if (t->mem) cudaFree(t->mem);
  if (t->tmem) cudaFree(t->tmem);
  if (t->rmem) cudaFree(t->rmem);
  if (t->gmem) cudaFree(t->gmem);
  if (t->plan) cudaFree(t->plan);
  delete t;
  return A1MPC_OK;
}

// ---- helpers -------------------------------------------------------------------------------
int a1mpc_device_alloc(a1mpc_handle* h, size_t bytes, void** ptr) {
  if (!h || !ptr) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  if (cudaMalloc(ptr, bytes) != cudaSuccess) { cudaGetLastError(); return fail(A1MPC_ENOMEM, "cudaMalloc failed"); }
  return A1MPC_OK;
}
int a1mpc_device_free(a1mpc_handle* h, void* ptr) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  CK(cudaFree(ptr));
  return A1MPC_OK;
}
int a1mpc_host_alloc(a1mpc_handle* h, size_t bytes, void** ptr) {
  if (!h || !ptr) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  if (cudaMallocHost(ptr, bytes) != cudaSuccess) { cudaGetLastError(); return fail(A1MPC_ENOMEM, "cudaMallocHost failed"); }
  return A1MPC_OK;
}
int a1mpc_host_free(a1mpc_handle* h, void* ptr) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaFreeHost(ptr));
  return A1MPC_OK;
}
int a1mpc_memcpy_h2d(a1mpc_handle* h, void* dst, const void* src, size_t bytes) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
  return A1MPC_OK;
}
int a1mpc_memcpy_d2h(a1mpc_handle* h, void* dst, const void* src, size_t bytes) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
  return A1MPC_OK;
}
static int join_gather(a1mpc_handle* h) {
  if (h->gather_pending) {   // the compute stream (and everything timed on it) waits for the outstanding collect
    CK(cudaStreamWaitEvent(h->stream, h->ev_gather_done, 0));
    h->gather_pending = false;
  }
  return A1MPC_OK;
}

int a1mpc_sync(a1mpc_handle* h) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  { int rc = join_gather(h); if (rc) return rc; }
  CK(cudaStreamSynchronize(h->stream));
  return A1MPC_OK;
}
int a1mpc_event_create(a1mpc_handle* h, void** ev) {
  if (!h || !ev) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  cudaEvent_t e;
  CK(cudaEventCreate(&e));
  *ev = (void*)e;
  return A1MPC_OK;
}
int a1mpc_event_destroy(a1mpc_handle* h, void* ev) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaEventDestroy((cudaEvent_t)ev));
  return A1MPC_OK;
}
int a1mpc_event_record(a1mpc_handle* h, void* ev) {
  if (!h || !ev) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  { int rc = join_gather(h); if (rc) return rc; }
  CK(cudaEventRecord((cudaEvent_t)ev, h->stream));
  return A1MPC_OK;
}
int a1mpc_event_elapsed_ms(a1mpc_handle* h, void* start, void* stop, float* ms) {
  if (!h || !start || !stop || !ms) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  CK(cudaEventSynchronize((cudaEvent_t)stop));
  CK(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
  return A1MPC_OK;
}
int64_t a1mpc_launch_count(const a1mpc_handle* h) { return h ? h->launches : 0; }

#if A1MPC_TIMELINE
// measurement build only (tools/timeline.py): device buffer of a1mpc::TL_CLASSES * (TL_CTAS + TL_QPS) * 4 u64 that the class kernels
// of every later solve write their CTA and QP records into (layout at tl_cta in a1mpc_device.cuh); NULL detaches it
int a1mpc_timeline_attach(a1mpc_handle* h, void* buf) {
  if (!h) return fail(A1MPC_EINVAL, "null handle");
  h->tl = static_cast<unsigned long long*>(buf);
  return A1MPC_OK;
}
#endif

int a1mpc_measure_fp64_peak(a1mpc_handle* h, double* tflops) {
  if (!h || !tflops) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  const int threads = 256, blocks = h->sm_count * 8, iters = 1 << 16;
  int rc;
  if ((rc = ensure_side(h, (size_t)threads * blocks * 8))) return rc;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  double best = 0.0;
  for (int rep = 0; rep < 4; ++rep) {
    CK(cudaEventRecord(e0, h->stream));
    fp64_peak_kernel<<<blocks, threads, 0, h->stream>>>((double*)h->d_side, iters);
    h->launches++;
    CK(cudaEventRecord(e1, h->stream));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    const double fl = 2.0 * 8.0 * (double)iters * threads * blocks;
    if (rep > 0) best = std::max(best, fl / (ms * 1e-3) * 1e-12);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *tflops = best;
  return A1MPC_OK;
}

int a1mpc_profile_begin(a1mpc_handle* h, int max_calls) {
  if (!h || max_calls <= 0) return fail(A1MPC_EINVAL, "bad argument");
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  while ((int)h->prof_ev.size() < max_calls * 8) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    h->prof_ev.push_back(e);
  }
  h->prof_cap = max_calls;
  h->prof_n = 0;
  h->prof_on = true;
  return A1MPC_OK;
}

int a1mpc_profile_end(a1mpc_handle* h, double* ms_per_class4, int* calls) {
  if (!h || !ms_per_class4) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < 4; ++k) ms_per_class4[k] = 0.0;
  for (int c = 0; c < h->prof_n; ++c)
    for (int k = 0; k < 4; ++k) {
      float ms = 0.f;
      CK(cudaEventElapsedTime(&ms, h->prof_ev[((size_t)c * 4 + k) * 2], h->prof_ev[((size_t)c * 4 + k) * 2 + 1]));
      ms_per_class4[k] += ms;
    }
  if (calls) *calls = h->prof_n;
  h->prof_on = false;
  return A1MPC_OK;
}

int a1mpc_flush_l2(a1mpc_handle* h) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  CK(cudaSetDevice(h->device));
  if (!h->d_flush) {
    h->flush_elems = 2 * h->l2_bytes / 8;  // twice the L2 (50 MB on an H100): every line of it is evicted
    if (cudaMalloc(&h->d_flush, h->flush_elems * 8) != cudaSuccess) { cudaGetLastError(); return fail(A1MPC_ENOMEM, "cudaMalloc failed"); }
  }
  flush_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(h->d_flush, h->flush_elems, 1.0);
  h->launches++;
  CK(cudaGetLastError());
  return A1MPC_OK;
}

/* ---- fused final collect over peer memory (one process per GPU, CUDA IPC) ------------------------------------------------ */
int a1mpc_peer_gather_create(a1mpc_handle* h, int nranks, int rank, int B_local, void* ipc_handle64) {
  if (!h || !ipc_handle64 || nranks < 1 || nranks > MAX_PEERS || rank < 0 || rank >= nranks || B_local <= 0) return fail(A1MPC_EINVAL, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t");
  CK(cudaSetDevice(h->device));
  a1mpc_peer_gather_destroy(h);
  auto& pg = h->peer;
  const size_t fbytes = (size_t)nranks * 12 * (size_t)B_local * 8;
  const size_t bytes = fbytes + (size_t)MAX_PEERS * 8 + 64;
  CK(cudaMalloc(&pg.local, bytes));
  CK(cudaMemset(pg.local, 0, bytes));
  pg.nranks = nranks; pg.rank = rank; pg.B = (size_t)B_local; pg.step = 0;
  pg.buf[rank] = (double*)pg.local;
  pg.flags[rank] = (unsigned long long*)((char*)pg.local + fbytes);
  cudaIpcMemHandle_t hd;
  CK(cudaIpcGetMemHandle(&hd, pg.local));
  std::memcpy(ipc_handle64, &hd, 64);
  return A1MPC_OK;
}

int a1mpc_peer_gather_connect(a1mpc_handle* h, const void* all_handles) {
  if (!h || !all_handles) return fail(A1MPC_EINVAL, "null argument");
  auto& pg = h->peer;
  if (!pg.local) return fail(A1MPC_EINVAL, "a1mpc_peer_gather_create first");
  CK(cudaSetDevice(h->device));
  const size_t fbytes = (size_t)pg.nranks * 12 * pg.B * 8;
  for (int p = 0; p < pg.nranks; ++p) {
    if (p == pg.rank) continue;
    cudaIpcMemHandle_t hd;
    std::memcpy(&hd, (const char*)all_handles + 64 * (size_t)p, 64);
    void* ptr = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(A1MPC_ECUDA, std::string("cudaIpcOpenMemHandle (rank ") + std::to_string(p) + "): " + cudaGetErrorString(e));
    pg.buf[p] = (double*)ptr;
    pg.flags[p] = (unsigned long long*)((char*)ptr + fbytes);
    pg.opened[p] = true;
  }
  pg.connected = true;
  return A1MPC_OK;
}

int a1mpc_peer_gather_buffer(a1mpc_handle* h, double** f_all) {
  if (!h || !f_all) return fail(A1MPC_EINVAL, "null argument");
  if (!h->peer.local) return fail(A1MPC_EINVAL, "a1mpc_peer_gather_create first");
  *f_all = (double*)h->peer.local;
  return A1MPC_OK;
}

int a1mpc_peer_gather_wait(a1mpc_handle* h) {
  if (!h) return fail(A1MPC_EINVAL, "null argument");
  auto& pg = h->peer;
  if (!pg.connected) return fail(A1MPC_EINVAL, "a1mpc_peer_gather_connect first");
  CK(cudaSetDevice(h->device));
  int* err = (int*)((char*)pg.local + (size_t)pg.nranks * 12 * pg.B * 8 + (size_t)MAX_PEERS * 8);
  // like the NCCL collect, the wait runs on the collect stream, forked after everything enqueued so far (this rank's signal included):
  // the next solve is not held back by a slower peer; a1mpc_sync / a1mpc_event_record join it.  (With the wait on the compute stream
  // every step ends in lock-step with the slowest rank.)
  cudaStream_t gs = (cudaStream_t)a1mpc_internal_gather_begin(h);
  if (!gs) return fail(A1MPC_ECUDA, "could not create the collect stream");
  // Preferred: stream memory operations (cuStreamWaitValue64, >=): the wait is done by the GPU's front end and occupies no SM.  A
  // spinning wait KERNEL sits on one SM for most of every step once the compute stream runs ahead, and since the persistent solve
  // kernels split their queue statically, one perturbed SM stretches the whole launch.  The kernel (polling every 5 us, ~2 s cap) remains as the fallback.
  typedef int (*wait_value_fn)(cudaStream_t, unsigned long long, unsigned long long, unsigned int);
  static wait_value_fn wait_value = nullptr;
  static bool looked_up = false;
  if (!looked_up) {
    looked_up = true;
    const char* ev = std::getenv("A1MPC_PEER_WAIT_KERNEL");
    if (!(ev && ev[0] == '1')) {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult qres;
      if (cudaGetDriverEntryPoint("cuStreamWaitValue64", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
        wait_value = (wait_value_fn)fn;
      else
        cudaGetLastError();
    }
  }
  bool done = false;
  if (wait_value) {
    done = true;
    for (int p = 0; p < pg.nranks && done; ++p)
      if (wait_value(gs, (unsigned long long)(uintptr_t)(pg.flags[pg.rank] + p), pg.step, 0u /* CU_STREAM_WAIT_VALUE_GEQ */) != 0) done = false;
    if (!done) { wait_value = nullptr; cudaGetLastError(); }   // not supported on this memory / driver: use the kernel from now on
    else h->launches += 0;
  }
  if (!done) {
    peer_wait_kernel<<<1, 32, 0, gs>>>(pg.flags[pg.rank], pg.nranks, pg.step, (long long)4e9 /* ~2 s */, err);
    h->launches++;
    CK(cudaGetLastError());
  }
  a1mpc_internal_gather_end(h);
  return A1MPC_OK;
}

int a1mpc_peer_gather_status(a1mpc_handle* h, int* timed_out_rank_plus_1) {
  if (!h || !timed_out_rank_plus_1) return fail(A1MPC_EINVAL, "null argument");
  auto& pg = h->peer;
  if (!pg.local) return fail(A1MPC_EINVAL, "a1mpc_peer_gather_create first");
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(timed_out_rank_plus_1, (char*)pg.local + (size_t)pg.nranks * 12 * pg.B * 8 + (size_t)MAX_PEERS * 8, sizeof(int), cudaMemcpyDeviceToHost));
  return A1MPC_OK;
}

int a1mpc_peer_gather_destroy(a1mpc_handle* h) {
  if (!h) return A1MPC_OK;
  auto& pg = h->peer;
  if (!pg.local) return A1MPC_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (int p = 0; p < MAX_PEERS; ++p) {
    if (pg.opened[p] && pg.buf[p]) cudaIpcCloseMemHandle(pg.buf[p]);
    pg.opened[p] = false; pg.buf[p] = nullptr; pg.flags[p] = nullptr;
  }
  cudaFree(pg.local);
  pg.local = nullptr; pg.connected = false; pg.nranks = 0; pg.B = 0;
  return A1MPC_OK;
}

}  // extern "C"

// accessors for a1mpc_nccl.cpp (which must not see the handle layout)
extern "C" {
void* a1mpc_internal_stream(a1mpc_handle* h) { return (void*)h->stream; }
// forks the collect stream off the compute stream (everything enqueued so far is visible to the collective) and returns it
void* a1mpc_internal_gather_begin(a1mpc_handle* h) {
  if (!h->gather_stream) {
    if (cudaStreamCreateWithFlags(&h->gather_stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    cudaEventCreateWithFlags(&h->ev_gather_in, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&h->ev_gather_done, cudaEventDisableTiming);
  }
  cudaEventRecord(h->ev_gather_in, h->stream);
  cudaStreamWaitEvent(h->gather_stream, h->ev_gather_in, 0);
  return (void*)h->gather_stream;
}
void a1mpc_internal_gather_end(a1mpc_handle* h) {
  cudaEventRecord(h->ev_gather_done, h->gather_stream);
  h->gather_pending = true;
}
int a1mpc_internal_device(a1mpc_handle* h) { return h->device; }
void** a1mpc_internal_nccl_slot(a1mpc_handle* h) { return &h->nccl_comm; }
void a1mpc_internal_set_error(const char* msg) { g_err = msg; }
}
