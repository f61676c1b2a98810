// emu_tick_rate.cpp -- the kernels of the multi-rate tick (a1mpc_tick_set_mpc_period) on the CPU block emulator of cuda_emu.h: the masked
// pack kernels and the unmasked ones they must agree with, tick_rate_kernel, tick_rate_reset_kernel and plan_forces_kernel.  TEST
// INFRASTRUCTURE ONLY: the unchanged device code, launched as a1mpc_api.cu launches it (thread per robot, 128-thread blocks), ld = B.
#define A1MPC_EMU 1
#include "cuda_emu.h"

#include "../../a1-qp-mpc-controller_b200/csrc/a1mpc_misc.cuh"

using namespace a1mpc;

namespace {
template <class F>
void launch(int B, F&& body) {
  const int pb = 128, pgrid = (B + pb - 1) / pb;
  for (int bx = 0; bx < pgrid; ++bx)
    a1emu::run_block(a1emu::Dim3{(unsigned)bx, 0, 0}, a1emu::Dim3{(unsigned)pgrid, 1, 1}, pb, 0, 0, body);
}
}  // namespace

extern "C" {

// REC_DOUBLES, REC_EXT_DOUBLES, WARM_HDR
void emu_rate_sizes(int* out) {
  out[0] = REC_DOUBLES;
  out[1] = REC_EXT_DOUBLES;
  out[2] = WARM_HDR;
}

// kind 0: pack_kernel (rec: 4 queues of cap records of REC_DOUBLES, count[1..4]); 1: warm_forget_no_contact_kernel (warm non-null) and
// pack_ext_kernel (rec: cap records of REC_EXT_DOUBLES, count[5]); 2: the same with pack_ext2_kernel (2 cap records, count[5] and [6]).
// runs non-null: the masked variant of each kernel with the run counters and the period.  sched, normals, iters, u_full, warm may be null.
int emu_rate_pack(int kind, int B, int horizon, const double* x0, const double* rot, const double* foot, const double* ref, const uint32_t* contact,
                  const uint32_t* sched, const double* normals, const uint32_t* runs, int period, double* rec, int cap, int* count, double* f_body,
                  int32_t* status, int32_t* iters, double* u_full, uint32_t* warm) {
  const DevInputs din{x0, rot, foot, ref, contact, (size_t)B, 0};
  DevOutputs dout{};
  dout.f_body = f_body; dout.status = status; dout.iters = iters; dout.u_full = u_full; dout.ld = (size_t)B; dout.f32 = 0;
  if (kind == 0) {
    if (runs) launch(B, [&]() { pack_due_kernel(din, B, rec, cap, count, dout, horizon, runs, period); });
    else launch(B, [&]() { pack_kernel(din, B, rec, cap, count, dout, horizon); });
    return 0;
  }
  if (warm) {
    if (runs) launch(B, [&]() { warm_forget_no_contact_due_kernel(din, sched, B, warm, horizon, runs, period); });
    else launch(B, [&]() { warm_forget_no_contact_kernel(din, sched, B, warm, horizon); });
  }
  if (kind == 1) {
    if (runs) launch(B, [&]() { pack_ext_due_kernel(din, sched, normals, B, rec, count, dout, horizon, runs, period); });
    else launch(B, [&]() { pack_ext_kernel(din, sched, normals, B, rec, count, dout, horizon); });
  } else {
    if (runs) launch(B, [&]() { pack_ext2_due_kernel(din, sched, normals, B, rec, cap, count, dout, horizon, runs, period); });
    else launch(B, [&]() { pack_ext2_kernel(din, sched, normals, B, rec, cap, count, dout, horizon); });
  }
  return 0;
}

// plan may be null (A1MPC_PLAYBACK_HOLD)
int emu_tick_rate(int B, int period, int horizon, uint32_t* runs, uint32_t* since, const double* rot, const double* plan, double* f_body) {
  launch(B, [&]() { tick_rate_kernel(B, period, horizon, runs, since, rot, plan, f_body); });
  return 0;
}

int emu_tick_rate_reset(int B, const uint8_t* mask, uint32_t* runs, uint32_t* since) {
  launch(B, [&]() { tick_rate_reset_kernel(B, mask, runs, since); });
  return 0;
}

int emu_plan_forces(int B, int horizon, const double* rot, const double* u_full, const uint32_t* step, double* f_body) {
  launch(B, [&]() { plan_forces_kernel(B, horizon, rot, u_full, step, f_body); });
  return 0;
}

}  // extern "C"
