// a1mpc_filter.cuh -- the moving-window filter of the device stages (a1mpc_swing.cuh, a1mpc_command.cuh), kept apart from their
// kernels so that both headers can use it from their own translation units.
#pragma once
#include "a1mpc_device.cuh"

namespace a1mpc {

// MovingWindowFilter::CalculateAverage (utils/filter.hpp:26-39) of window W: once the window is full the oldest value is subtracted
// BEFORE the new one is added, both by Neumaier's compensated sum, and the average always divides by the full window size (biased
// towards 0 while filling).  The window of the robot whose state starts at s (stride ld): slots at rows vals.., sum, correction,
// fill count and ring head at rows hdr..hdr+3.  The one filter of every device stage (sw_filter of a1mpc_swing.cuh, the IMU filters of
// a1mpc_command.cuh).
__device__ __forceinline__ void sw_neumaier(double& sum, double& corr, double v) {
  const double ns = sum + v;
  if (fabs(sum) >= fabs(v)) corr += (sum - ns) + v;
  else corr += (v - ns) + sum;
  sum = ns;
}
__device__ __forceinline__ double mw_filter(double* s, size_t ld, int W, int vals, int hdr, double x) {
  double* val = s + (size_t)vals * ld;
  double* hd = s + (size_t)hdr * ld;
  double sum = hd[0], corr = hd[ld];
  int cnt = (int)hd[2 * ld], head = (int)hd[3 * ld];
  if (cnt < W) {
    val[(size_t)cnt * ld] = x;
    ++cnt;
  } else {
    sw_neumaier(sum, corr, -val[(size_t)head * ld]);
    val[(size_t)head * ld] = x;
    head = head + 1 == W ? 0 : head + 1;
  }
  sw_neumaier(sum, corr, x);
  hd[0] = sum; hd[ld] = corr; hd[2 * ld] = (double)cnt; hd[3 * ld] = (double)head;
  return (sum + corr) / (double)W;
}

}  // namespace a1mpc
